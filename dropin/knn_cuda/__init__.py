"""H100 drop-in for ``knn_cuda``: ``KNN(k=1, transpose_mode=True)``, the only form the BUFFER-X reference uses
(models/BUFFERX.py:481,486,511), on bufferx_b200's ``bx_knn1`` kernel, forward only.

``KNN(k=1, transpose_mode=True)(ref [B,Nr,D], query [B,Nq,D]) -> (dist [B,Nq,1] float32, idx [B,Nq,1] int64)``: for each
query row the first ref row (in ref order) with the smallest squared distance, summed over D in order without FMA;
dist = sqrtf of it.  Needs the repository root on ``sys.path`` as well (it imports ``bufferx_b200.ops``).
"""
import torch

from bufferx_b200 import ops
from bufferx_b200.ops import BufferXError

__all__ = ["KNN"]


class KNN(torch.nn.Module):
    def __init__(self, k, transpose_mode=False):
        super().__init__()
        if k != 1 or not transpose_mode:
            raise NotImplementedError(f"knn_cuda.KNN: only KNN(k=1, transpose_mode=True) is supported, got k={k}, "
                                      f"transpose_mode={transpose_mode}")
        self.k, self.transpose_mode = k, transpose_mode

    def forward(self, ref, query):
        ref = ops.dropin_tensor(ref, "ref", "[B,Nr,D]")
        query = ops.dropin_tensor(query, "query", "[B,Nq,D]")
        if ref.shape[0] != query.shape[0] or ref.shape[2] != query.shape[2] or ref.device != query.device:
            raise BufferXError(f"KNN: expected ref [B,Nr,D] and query [B,Nq,D] on one device, got {tuple(ref.shape)} on {ref.device} "
                               f"and {tuple(query.shape)} on {query.device}")
        if ref.shape[1] == 0:
            raise BufferXError("KNN: ref has no rows")
        with torch.cuda.device(ref.device):
            dist, idx = ops.knn1(ref, query)
        return dist.unsqueeze(2), idx.unsqueeze(2)
