"""The C oracle's FPS at the sizes only the grid-wide kernel (bx_fps_large) runs, N > 524288, where the GPU tests hold
that kernel to it bit for bit: teacher-forced against the float64 restatement of pointnet2's furthest_point_sample
(oracle.fps_fp64, bounds derived in tests/test_frontend_fp64_cpu.py), and equal to a vectorised restatement of the
upstream 512-thread block reduction, which pins the tie rule the float64 check leaves open."""
import numpy as np
import pytest

from oracle import frontend_cases as F
from oracle.frontend_cases import merge, report

F32 = np.float32


def _fps_block_reduction(xyz, m, bs=512):
    """pointnet2's kernel with bs threads: thread t scans k = t, t + bs, ... keeping its first strict maximum, then the
    tree reduction keeps the lower position unless the upper one is strictly larger.  fp32 arithmetic, no FMA."""
    n = len(xyz)
    x, y, z = (xyz[:, i].astype(F32) for i in range(3))
    mag = ((x * x) + (y * y)) + (z * z)
    valid = mag.astype(np.float64) > 1e-3
    rows = -(-n // bs)
    temp = np.full(n, 1e10, F32)
    idx, old = [0], 0
    for _ in range(1, m):
        dx, dy, dz = x - x[old], y - y[old], z - z[old]
        temp = np.minimum(temp, ((dx * dx) + (dy * dy)) + (dz * dz))
        v = np.full(rows * bs, -1.0, F32)
        v[:n] = np.where(valid, temp, F32(-1.0))
        v = v.reshape(rows, bs)                      # column t = thread t's points in scan order
        col = v.argmax(0)                            # first maximum of each thread
        best, besti = v[col, np.arange(bs)], col * bs + np.arange(bs)
        s = bs // 2
        while s >= 1:
            up = best[s:2 * s] > best[:s]
            best[:s] = np.where(up, best[s:2 * s], best[:s])
            besti[:s] = np.where(up, besti[s:2 * s], besti[:s])
            s //= 2
        old = int(besti[0]) if best[0] >= 0 else 0
        idx.append(old)
    return np.array(idx, np.int32)


def test_block_reduction_restatement_matches_small_oracle(oracle):
    """The restatement itself, where the per-thread reference of tests/test_oracle_cpu.py runs: duplicates and lattice
    ties at bs = 512."""
    for kind in ("dup", "lattice"):
        xyz = F.fps_cloud(kind, 3000, seed=5)
        assert np.array_equal(_fps_block_reduction(xyz, 48), oracle.fps(xyz, 48)), kind


@pytest.mark.parametrize("n", [524289, 1048576])
@pytest.mark.parametrize("kind,offset", [("uniform", 1e4), ("dup", 0.0), ("lattice", 0.0), ("fewvalid", 0.0)])
def test_fps_oracle_beyond_the_cluster_limit(oracle, n, kind, offset):
    xyz = F.fps_cloud(kind, n, seed=n % 97, offset=offset, k_valid=40)
    idx = oracle.fps(xyz, 64)
    acc = F.check_fps(xyz, 64, idx)
    assert np.array_equal(idx, _fps_block_reduction(xyz, 64)), "oracle differs from the block reduction"
    report(f"fps oracle n={n} {kind} offset {offset:g}", merge({}, acc))
