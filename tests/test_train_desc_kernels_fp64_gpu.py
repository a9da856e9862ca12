"""GPU: every wrapper of the Desc training step's kernels (csrc/bx_train_desc.cu) called directly and held to the derived
float64 bounds of oracle/train_desc_cases.py, at the shapes where tiling and reductions go wrong (fewer rows than the 64
reduction splits, rows at the split boundaries, one live channel padded to four) and on edge inputs: the ReLU boundary of
the pool layer's BatchNorms, L2 norms of exactly 1e-12, all-dead voxels and NaN at the cylindrical raster's seams."""
import numpy as np
import pytest
import torch

from oracle import train_desc_cases as D
from oracle.train_step_cases import from_blocked, merge, report, to_blocked

pytestmark = pytest.mark.gpu
F64 = torch.float64


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def _ops():
    from bufferx_b200 import ops
    return ops


def _g(a, dev, dtype=F64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev, dtype)


def _blk(a, dev):
    return _g(to_blocked(np.asarray(a, np.float64)), dev)


def _unblk(t):
    return from_blocked(t.cpu().numpy())


# ------------------------------------------------------------------------------------------------ conv1x1 (float64)
@pytest.mark.parametrize("n", [1, 2, 65])
@pytest.mark.parametrize("shape", D.CONV1X1_SHAPES)
def test_conv1x1_float64(dev, shape, n):
    ops = _ops()
    Cin, Cout = shape
    res = {}
    for S in (1, 139, 140):
        x, w, b, out0 = D.conv1x1_case(n, Cin, Cout, S, seed=Cin + Cout + S + n, live=1 if shape == (16, 4) else None,
                                       live_in=1 if shape == (4, 16) else None)
        xb, wg, bg = _blk(x, dev), _g(w, dev), _g(b, dev)
        merge(res, D.check_conv1x1(x, w, b, _unblk(ops.conv1x1(xb, wg, bg))))
        merge(res, D.check_conv1x1(x, w, None, _unblk(ops.conv1x1(xb, wg))))
        ob = _blk(out0, dev)
        r = ops.conv1x1(xb, wg, bg, out=ob)
        assert r.data_ptr() == ob.data_ptr()
        merge(res, D.check_conv1x1(x, w, b, _unblk(ob), out0=out0))
    report(f"conv1x1_f64 {Cin}->{Cout} n={n}", res)


# ------------------------------------------------------------------------------------------------ cross_sums
@pytest.mark.parametrize("C", D.CROSS_C)
@pytest.mark.parametrize("nS", D.CROSS_NS)
def test_cross_sums(dev, nS, C):
    ops = _ops()
    n, S = nS
    res = {}
    for kind in ("offset",) if n * S > 140 else ("offset", "const", "random"):
        X, Dm = D.cross_case(n, C[0], C[1], S, kind, seed=n + S)
        Xb, Db = _blk(X, dev), _blk(Dm, dev)
        got = ops.cross_sums(Xb, Db)
        merge(res, D.check_cross_sums(X, Dm, got.cpu().numpy()))
        assert torch.equal(got, ops.cross_sums(Xb, Db)), "cross_sums is not bit-identical across calls"
    report(f"cross_sums {C} n={n} S={S}", res)


# ------------------------------------------------------------------------------------------------ bn_backward
@pytest.mark.parametrize("n", D.BNA_N)
@pytest.mark.parametrize("C", [16, 4])
def test_bn_backward_mask_is_the_forwards(dev, C, n):
    """The pool layer's BatchNorm + ReLU backward: the forward is ops.bn_apply on the folded (scale, shift), as
    MiniSpinNet.train_desc runs it; z within 8 ulp of each boundary channel's root.  C = 4 is the attention's BN(1)
    padded to four channels with all-zero parameters."""
    ops = _ops()
    S = 140
    dy, z, mean, rstd, gam, _, scale, shift = D.bna_case(n, C, S, seed=n + C, pad=C == 4)
    zb = _blk(z, dev)
    yb = ops.bn_apply(zb, _g(scale, dev), _g(shift, dev), True)
    y = _unblk(yb)
    assert np.array_equal(y, D.fwd_relu(z, scale, shift)), "bn_apply is not one fused multiply-add"
    dx, sums = ops.bn_backward(_blk(dy, dev), zb, yb, *(_g(t, dev) for t in (mean, rstd, gam)))
    res = D.check_bn_affine_backward(dy, z, y, mean, rstd, gam, _unblk(dx), sums.cpu().numpy())
    report(f"bn_affine_backward C={C} n={n}", res)


# ------------------------------------------------------------------------------------------------ point layer
PNT = [(1, 1, 1, 0.0), (2, 1, 2, 0.0), (1, 420, 10, 0.0), (1, 420, 255, 0.0), (65, 420, 2, 0.0), (65, 1, 255, 0.0),
       (2, 420, 10, 10.0), (2, 420, 10, 1e3)]


@pytest.mark.parametrize("K,V,nv,offset", PNT)
def test_point_layer_against_derived_bounds(dev, K, V, nv, offset):
    ops = _ops()
    inv, W, b, gam, beta = D.pnt_case(K, V, nv, offset, seed=K + V + nv)
    mean, rstd, scale, shift = D.pnt_stats(inv, W, b, gam, beta)
    ig = _g(inv, dev, torch.float32)
    feat, arg = ops.pnt_forward(ig, _g(W, dev), _g(b, dev), _g(scale, dev), _g(shift, dev))
    fc = _unblk(feat)
    res = D.check_pnt_forward(inv, W, b, scale, shift, fc, arg.cpu().numpy())
    if K * V * nv >= 20:
        assert (fc[0, 0, 0] == 0) and int(arg[0, 0, 0]) == 0, "the all-dead voxel: feat 0 from its first sample"
    dfeat = np.random.default_rng(K + nv).normal(size=(K, 16, V))
    out = ops.pnt_backward(ig, arg, _blk(dfeat, dev), _g(W, dev), _g(b, dev), _g(mean, dev), _g(rstd, dev), _g(gam, dev),
                           _g(scale, dev), _g(shift, dev), ops.moments3(ig))
    merge(res, D.check_pnt_backward(inv, arg.cpu().numpy(), fc, dfeat, W, b, mean, rstd, gam, out.cpu().numpy()))
    report(f"point layer K={K} V={V} nv={nv} offset={offset}", res)


def test_point_layer_backward_mask_at_the_relu_boundary(dev):
    """A selected sample at the ReLU boundary, probed with a one-hot dfeat: dbeta is exactly 1 where the forward's feat is
    > 0 and exactly 0 where it is 0."""
    ops = _ops()
    inv, W, b, scale, shift, mean, rstd, gam = D.pnt_boundary_case()
    ig = _g(inv, dev, torch.float32)
    args = [_g(t, dev) for t in (W, b)]
    feat, arg = ops.pnt_forward(ig, *args, _g(scale, dev), _g(shift, dev))
    fc = _unblk(feat)
    mo = ops.moments3(ig)
    live = 0
    for c in range(16):
        df = np.zeros((2, 16, 8))
        df[0, c, 0] = 1.0
        out = ops.pnt_backward(ig, arg, _blk(df, dev), *args, _g(mean, dev), _g(rstd, dev), _g(gam, dev), _g(scale, dev),
                               _g(shift, dev), mo).cpu().numpy()
        want = 1.0 if fc[0, c, 0] > 0 else 0.0
        live += int(want)
        assert out[c, 5] == want, f"channel {c}: dbeta {out[c, 5]!r}, the forward's feat {fc[0, c, 0]!r}"
    print(f"\n[train-desc-fp64] point-layer boundary: {live} of 16 boundary samples passed the ReLU")


# ------------------------------------------------------------------------------------------------ pool layer
@pytest.mark.parametrize("K", [1, 2, 65])
def test_pool_layer_at_the_normalisation_eps(dev, K):
    ops = _ops()
    x, w = D.pool_case(K, seed=K)
    wb = np.zeros((K, 1, 140, 4))
    wb[:, 0, :, 0] = w
    xg, wg = _blk(x, dev), _g(wb, dev)
    f, desc, equi = ops.pool_forward(xg, wg)
    fc = f.cpu().numpy()
    assert fc[0, 3] == D.EPS and np.count_nonzero(fc[0]) == 1, "f of patch 0 is not [.., 1e-12, ..]"
    res = D.check_pool_forward(x, w, fc, desc.cpu().numpy(), equi.cpu().numpy().reshape(K, 32, 140))
    rng = np.random.default_rng(K)
    ddesc = rng.normal(size=(K, 32)).astype(np.float32)
    dequi = rng.normal(size=(K, 32, 7, 20)).astype(np.float32)
    for fv in (fc, D.pool_f_cases(K, seed=K)):           # the forward's f, then f of norm 1e-12, +-1 ulp and 0
        dx, dw = ops.pool_backward(xg, wg, _g(fv, dev), _g(ddesc, dev, torch.float32), _g(dequi, dev, torch.float32))
        dwc = dw.cpu().numpy()
        assert (dwc[:, 0, :, 1:] == 0).all()
        merge(res, D.check_pool_backward(x, w, fv, ddesc, dequi, _unblk(dx), dwc[:, 0, :, 0]))
    report(f"pool layer K={K}", res)


# ------------------------------------------------------------------------------------------------ cylindrical convolution
@pytest.mark.parametrize("where", ["x", "dy"])
@pytest.mark.parametrize("ea", [(0, 0), (6, 19), (3, 10)])
@pytest.mark.parametrize("Din", [1, 3])
def test_cyl_nan_footprint(dev, Din, ea, where):
    """One NaN in x (at depth slice Din - 1) or in dy: out, dx and dW NaN exactly where float64 F.conv3d on the padded
    input has them -- the azimuth seam 19 <-> 0 wraps, elevation is zero padded, the data gradient's taps are flipped."""
    ops = _ops()
    n, Cin, Cout = 2, 16, 16
    x5, w, b, dy = D.cyl_case(n, Cin, Cout, Din, seed=Din + ea[0])
    if where == "x":
        x5[1, 5, Din - 1, ea[0], ea[1]] = np.nan
    else:
        dy[1, 9, ea[0], ea[1]] = np.nan
    xb = _blk(x5.reshape(n, Cin, Din * 140), dev)
    Wt = _g(np.ascontiguousarray(w.reshape(Cout, Cin, -1).transpose(2, 1, 0)), dev)
    out = ops.cyl_forward(xb, Wt, _g(b, dev), Din)
    dx, dW = ops.cyl_backward(xb, _blk(dy.reshape(n, Cout, 140), dev), Wt, Din)
    res = D.check_cyl(x5, w, b, dy, _unblk(out).reshape(n, Cout, 7, 20), _unblk(dx).reshape(x5.shape),
                      dW.cpu().numpy().transpose(2, 1, 0).reshape(w.shape))
    report(f"cyl NaN Din={Din} {where}@{ea}", res)
