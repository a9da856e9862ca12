"""CPU check of the coverage argument of the hash-grid patch gathering (csrc/bx_patches.cu, hg_coord / hg_inv_cell /
hg_window): a point that the kernel's fp32 test d2 < r*r accepts lies in a cell of the key-point's query window -- in fp32,
with the kernel's own arithmetic (cell edge 1.001 * radius, cell value a = fl(v * fl(1 / fl(r * 1.001))), cell floor(a),
window [floor(fl(a - w)), floor(fl(a + w))] with w = 0.9993 + 2^-22 |a|).  Near the origin that is the key-point's cell +-1;
far from it the fp32 spacing of the cell values grows and a hit can land two cells away where a crosses a power of two, which
the window covers.  The GPU tests (test_select_patches_grid_equals_scan, tests/test_frontend_fp64_gpu.py) compare whole
results; this pins the bound."""
import numpy as np
import pytest

F32 = np.float32


def _ic(r):
    return F32(1.0) / (F32(r) * F32(1.001))


def _cell_value(v, r):
    return (np.asarray(v, F32) * _ic(r)).astype(F32)


def _window(a):
    a = np.asarray(a, F32)
    w = (F32(0.9993) + (F32(2.0 ** -22) * np.abs(a)).astype(F32)).astype(F32)
    lo = np.floor((a - w).astype(F32)).astype(np.int64)
    hi = np.floor((a + w).astype(F32)).astype(np.int64)
    return lo, hi


def _hits(q, p, radius):
    dx, dy, dz = (q[:, 0] - p[:, 0]), (q[:, 1] - p[:, 1]), (q[:, 2] - p[:, 2])
    d2 = ((dx * dx).astype(F32) + (dy * dy).astype(F32)).astype(F32) + (dz * dz).astype(F32)
    return d2.astype(F32) < F32(radius) * F32(radius)


def _pairs(radius, centre, extent, n, seed):
    """Key points uniform in centre +- extent (per axis), points just inside the radius in random and axis directions."""
    rng = np.random.default_rng(seed)
    q = (centre + rng.uniform(-extent, extent, size=(n, 3))).astype(F32)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d[: n // 2] = np.eye(3)[rng.integers(0, 3, n // 2)] * rng.choice([-1.0, 1.0], size=(n // 2, 1))
    p = (q.astype(np.float64) + d * rng.uniform(0.9, 1.0, size=(n, 1)) * radius).astype(F32)
    return q, p


def _check(q, p, radius):
    hit = _hits(q, p, radius)
    a, b = _cell_value(q, radius), _cell_value(p, radius)
    lo, hi = _window(a)
    cell = np.floor(b).astype(np.int64)
    inside = (cell >= lo) & (cell <= hi)
    assert inside[hit].all(), f"a hit outside the key point's window: {np.argwhere(hit[:, None] & ~inside)[:4]}"
    return hit, hi - lo + 1, a


@pytest.mark.parametrize("radius,extent", [(0.05, 3.0), (0.3, 60.0), (1.5, 120.0), (0.0123, 50.0), (2.0, 8000.0)])
def test_neighbour_within_radius_is_within_one_cell(radius, extent):
    """Up to 4096 cells per axis a hit is also within one cell of its key point's (the classic query's coverage)."""
    q, p = _pairs(radius, 0.0, extent, 400000, int(radius * 1e4) + int(extent))
    hit, n, a = _check(q, p, radius)
    assert hit.mean() > 0.5 and n.max() <= 4 and (n[(np.abs(a) < 2900).all(1)] <= 3).all()
    assert extent / (radius * 1.001) <= 4096.0
    dc = np.abs(np.floor(a).astype(np.int64) - np.floor(_cell_value(p, radius)).astype(np.int64))
    assert dc[hit].max() <= 1, f"a hit {dc[hit].max()} cells away from its key-point"


# clouds straddling the power-of-two cell values 2^13 .. 2^20, where the classic cell +-1 query loses neighbours
STRADDLE = [(r, k) for k in (13, 16, 17, 18, 19, 20) for r in (0.05, 0.09, 0.3, 0.77)]


@pytest.mark.parametrize("radius,k", STRADDLE)
def test_window_covers_power_of_two_cell_boundaries(radius, k):
    centre = 2.0 ** k * float(F32(F32(radius) * F32(1.001)))         # the cloud's cell values straddle 2^k
    q, p = _pairs(radius, centre, 4 * radius, 200000, k * 100 + int(radius * 100))
    hit, n, a = _check(q, p, radius)
    assert hit.mean() > 0.5 and n.max() <= 4
    sgn = -1.0
    q2, p2 = q * F32(sgn), p * F32(sgn)                                # and the negative side
    _check(q2, p2, radius)


def test_classic_query_loses_these_neighbours():
    """Two hits two cells away from their key point (cells 131071 / 131073 and 262143 / 262145): the +-1 cell query of
    earlier versions missed them; the window takes them."""
    for r, qx, px in ((0.09, 11808.27734375, 11808.3671875), (0.05, 13120.3076171875, 13120.357421875)):
        q = np.array([[qx, 0.0, 0.0]], F32)
        p = np.array([[px, 0.0, 0.0]], F32)
        assert _hits(q, p, r)[0]
        a, b = _cell_value(q, r)[0, 0], _cell_value(p, r)[0, 0]
        assert int(np.floor(b)) - int(np.floor(a)) == 2
        _check(q, p, r)


def test_window_size_bounds():
    """At most 3 cells per axis below ~2900 cells from the origin, at most 4 below 2^21 (the kernel's 64-bucket loop); the
    kernel scans the whole cloud beyond that."""
    a = np.concatenate([np.linspace(-2900, 2900, 2_000_001), np.linspace(-2.0 ** 21 + 1, 2.0 ** 21 - 1, 2_000_001)]).astype(F32)
    lo, hi = _window(a)
    n = hi - lo + 1
    assert (n[: 2_000_001] <= 3).all() and (n <= 4).all() and (n >= 2).all()
