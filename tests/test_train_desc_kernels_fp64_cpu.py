"""The Desc training step's kernel checks (oracle/train_desc_cases.py) without a GPU: each accepts a float64 restatement of
its kernel in csrc/bx_train_desc.cu (the same split order, mask, tap walk and padding) and rejects a subtly wrong one.
tests/test_train_desc_kernels_fp64_gpu.py holds the kernels to the same checks."""
import math

import numpy as np
import pytest

from oracle import train_desc_cases as D
from oracle import train_step_cases as TS
from oracle.train_step_cases import fma64


# ------------------------------------------------------------------------------------------------ restatements
def emu_conv1x1(x, w, b, out0=None, mutation=None):
    n, Cin, S = x.shape
    acc = np.broadcast_to((np.zeros(w.shape[1]) if b is None else b)[None, :, None], (n, w.shape[1], S)).copy()
    for ci in range(Cin):
        acc = fma64(w[ci][None, :, None], x[:, ci:ci + 1], acc)
    return acc if out0 is None or mutation == "out_ignored" else out0 + acc


def emu_cross_sums(X, Dm, mutation=None):
    n, Ca, S = X.shape
    Xr, Dr = X.transpose(1, 0, 2).reshape(Ca, -1), Dm.transpose(1, 0, 2).reshape(Dm.shape[1], -1)
    R = n * S
    per = math.ceil(R / D.SPLITS)
    out = np.zeros((Ca, Dm.shape[1]))
    for s in range(D.SPLITS):
        if mutation == "drop_split" and s == min(D.SPLITS - 1, (R - 1) // per):
            continue
        out += Xr[:, s * per:(s + 1) * per] @ Dr[:, s * per:(s + 1) * per].T
    return out.T.copy() if mutation == "transposed" else out


def emu_bn_affine_backward(dy, z, y, mean, rstd, gam, beta, mutation=None):
    n, C, S = z.shape
    xh = (z - mean[None, :, None]) * rstd[None, :, None]
    if mutation == "unfolded_mask":                    # the former mask: gamma x^ + beta > 0, unfused
        keep = gam[None, :, None] * xh + beta[None, :, None] > 0
    elif mutation == "unfolded_mask_fma":              # the same, as nvcc contracts it: fma(gamma, x^, beta) > 0
        keep = fma64(gam[None, :, None], xh, beta[None, :, None]) > 0
    elif mutation == "mask_ge":                        # >= for >: also keeps the forward's exact zeros before the ReLU
        G = gam * rstd
        keep = fma64(z, G[None, :, None], (beta - mean * G)[None, :, None]) >= 0
    else:
        keep = y > 0
    dz = np.where(keep, dy, 0.0)
    s0, s1 = dz.sum(axis=(0, 2)), (dz * xh).sum(axis=(0, 2))
    N = n * S
    m2 = 0.0 if mutation == "no_xh_m2" else (s1 / N)[None, :, None]
    dx = (gam * rstd)[None, :, None] * ((dz - (s0 / N)[None, :, None]) - xh * m2)
    return dx, np.stack([s0, s1])


def emu_pnt_forward(inv, W, b, scale, shift, mutation=None):
    y = D._pnt_y(inv, W, b)
    r = np.maximum(fma64(y, scale, shift), 0.0)          # [K, V, nv, 16]
    if mutation == "last_max":
        arg = r.shape[2] - 1 - r[:, :, ::-1].argmax(2)
    else:
        arg = r.argmax(2)
    return r.max(2).transpose(0, 2, 1), arg.transpose(0, 2, 1)


def emu_pnt_backward(inv, arg, feat, dfeat, W, b, mean, rstd, gam, mutation=None):
    K, V, nv, _ = inv.shape
    x = inv.astype(np.float64)
    kk, cc, vv = np.meshgrid(np.arange(K), np.arange(16), np.arange(V), indexing="ij")
    xs = x[kk, vv, arg]                                   # [K, 16, V, 3] the selected samples
    y = np.einsum("kcvj,cj->kcv", xs, W) + b[None, :, None]
    dz = np.where(feat > 0, dfeat, 0.0)
    xh = (y - mean[None, :, None]) * rstd[None, :, None]
    S0, S1 = dz.sum((0, 2)), (dz * xh).sum((0, 2))
    Sj = np.einsum("kcv,kcvj->cj", dz, xs)
    xr = x.reshape(-1, 3)
    R = xr.shape[0] if mutation != "R_without_zero_slots" else int((xr != 0).any(1).sum())
    mo, M = xr.sum(0), xr.T @ xr
    m1, m2, G, off = S0 / R, S1 / R, gam * rstd, b - mean
    sxh = rstd * (W @ mo + R * off)
    sxi = rstd[:, None] * (W @ M + off[:, None] * mo[None])
    out = np.empty((16, 6))
    out[:, :3] = G[:, None] * (Sj - m1[:, None] * mo[None] - m2[:, None] * sxi)
    out[:, 3] = G * (S0 - R * m1 - m2 * sxh)
    out[:, 4], out[:, 5] = S1, S0
    return out


def _normalize_bwd(v, g, eps, mutation):
    n = np.sqrt((v * v).sum(0))
    big = n > eps if mutation == "strict_gt" else n >= eps
    den = np.where(big, n, eps)
    y = v / den
    yg = (y * g).sum(0)
    return np.where(big, (g - y * yg) / den, g / eps)


def emu_pool_forward(x, w, mutation=None):
    P = 139 if mutation == "avg_139" else 140
    f = (x[:, :, :P] * w[:, None, :P]).sum(2) / P
    desc = f / np.maximum(np.sqrt((f * f).sum(1, keepdims=True)), D.EPS)
    equi = x / np.maximum(np.sqrt((x * x).sum(1, keepdims=True)), D.EPS)
    return f, desc.astype(np.float32), equi.astype(np.float32)


def emu_pool_backward(x, w, f, ddesc, dequi, mutation=None):
    K = x.shape[0]
    df = _normalize_bwd(f.T, ddesc.astype(np.float64).T, D.EPS, mutation).T
    de = np.stack([_normalize_bwd(x[k], dequi[k].reshape(32, 140).astype(np.float64), D.EPS, mutation) for k in range(K)])
    return de + df[:, :, None] * w[:, None, :] / 140, (df[:, :, None] * x).sum(1) / 140


def _src(e, a, de, da, mutation):
    ee, aa = e + de - 1, a + da - 1
    if mutation == "wrap_elevation":
        ee %= D.CYL_E
    elif not 0 <= ee < D.CYL_E:
        return None
    if mutation == "wrap_one_side":
        if aa >= D.CYL_A:
            return None
        aa %= D.CYL_A
    else:
        aa %= D.CYL_A
    return ee, aa


def _gather(x, mutation):
    """x [n, C, 7, 20] -> [9, n, C, 7, 20]: the loader's value of tap (de, da) at every output position (0 outside)."""
    out = np.zeros((9,) + x.shape)
    for t in range(9):
        de, da = t // 3, t % 3
        for e in range(D.CYL_E):
            for a in range(D.CYL_A):
                s = _src(e, a, de, da, mutation)
                if s is not None:
                    out[t, :, :, e, a] = x[:, :, s[0], s[1]]
    return out


def emu_cyl(x5, w, b, dy, mutation=None):
    """out, dx, dW as bx_td_cyl_forward / dgrad / wgrad compute them (dgrad: the same loader on dy, taps flipped)."""
    n, Cin, Din = x5.shape[:3]
    Cout = w.shape[0]
    wt = w.reshape(Cout, Cin, Din, 9)
    out = np.broadcast_to(b[None, :, None, None], (n, Cout, 7, 20)).copy()
    gx = [_gather(x5[:, :, d], mutation) for d in range(Din)]
    for d in range(Din):
        out += np.einsum("tncea,oct->noea", gx[d], wt[:, :, d])
    gdy = _gather(dy, mutation)
    dx = np.zeros(x5.shape)
    for d in range(Din):
        taps = np.arange(9) if mutation == "dgrad_unflipped" else 8 - np.arange(9)
        dx[:, :, d] = np.einsum("tnoea,oct->ncea", gdy, wt[:, :, d][:, :, taps])
    R = n * 140
    per = math.ceil(R / D.SPLITS)
    dW = np.zeros_like(wt)
    for d in range(Din):
        X = gx[d].reshape(9, n, Cin, 140).transpose(0, 2, 1, 3).reshape(9, Cin, R)
        Y = dy.reshape(n, Cout, 140).transpose(1, 0, 2).reshape(Cout, R)
        for s in range(D.SPLITS):
            if mutation == "wgrad_drop_split" and s == (R - 1) // per:
                continue
            sl = slice(s * per, (s + 1) * per)
            dW[:, :, d] += np.einsum("tcr,or->oct", X[:, :, sl], Y[:, sl])
    return out, dx, dW.reshape(w.shape)


# ------------------------------------------------------------------------------------------------ tests
def test_conv1x1_check_accepts_the_kernel_and_rejects_an_ignored_out():
    for (Cin, Cout) in [(32, 16), (16, 4), (4, 16)]:
        x, w, b, out0 = D.conv1x1_case(2, Cin, Cout, 139, seed=Cin, live=1 if Cout == 4 else None)
        D.check_conv1x1(x, w, b, emu_conv1x1(x, w, b))
        D.check_conv1x1(x, w, None, emu_conv1x1(x, w, None))
        D.check_conv1x1(x, w, b, emu_conv1x1(x, w, b, out0), out0=out0)
        with pytest.raises(AssertionError):
            D.check_conv1x1(x, w, b, emu_conv1x1(x, w, b, out0, "out_ignored"), out0=out0)


@pytest.mark.parametrize("mutation", ["drop_split", "transposed"])
def test_cross_sums_check_rejects(mutation):
    for n, S in [(1, 65), (1, 140), (4, 140)]:
        X, Dm = D.cross_case(n, 4, 4, S, "offset", seed=S)
        D.check_cross_sums(X, Dm, emu_cross_sums(X, Dm))
        with pytest.raises(AssertionError):
            D.check_cross_sums(X, Dm, emu_cross_sums(X, Dm, mutation))


@pytest.mark.parametrize("mutation", ["unfolded_mask", "unfolded_mask_fma"])
@pytest.mark.parametrize("C", [16, 4])
def test_bn_affine_backward_check_rejects_the_unfolded_mask(C, mutation):
    """The forward's mask y > 0 of y = fma(z, scale, shift) and the former kernel's gamma ((z - mean) rstd) + beta > 0
    (unfused, or fused as nvcc contracts it by default) round to opposite signs on some of the inputs within 8 ulp of the
    boundary."""
    flips = 0
    for n in (2, 65):
        dy, z, mean, rstd, gam, beta, scale, shift = D.bna_case(n, C, 140, seed=n + C, pad=C == 4)
        y = D.fwd_relu(z, scale, shift)
        D.check_bn_affine_backward(dy, z, y, mean, rstd, gam, *emu_bn_affine_backward(dy, z, y, mean, rstd, gam, beta))
        dx, sums = emu_bn_affine_backward(dy, z, y, mean, rstd, gam, beta, mutation)
        f = int((dx != emu_bn_affine_backward(dy, z, y, mean, rstd, gam, beta)[0]).any(axis=(0, 2)).sum())
        flips += f
        if f:
            with pytest.raises(AssertionError, match="ReLU mask"):
                D.check_bn_affine_backward(dy, z, y, mean, rstd, gam, dx, sums)
    assert flips > 0


@pytest.mark.parametrize("mutation", [None, "mask_ge", "no_xh_m2"], ids=["restatement", "mask_ge", "no_xh_m2"])
def test_bn_backward_check_at_gamma_1(mutation):
    """gamma = 1, the affine = False BatchNorms of CostNet and Cylindrical_Net (rstd = scale, y = bn_apply's
    fma(z, scale, shift) with ReLU), on train_step_cases.mask_case: x^ exactly 0 and +-1 ulp, dead and constant channels.
    The check accepts the restatement and, on every shape, rejects a mask that also keeps the forward's exact zeros and a
    dx without x^ m2."""
    for n, S in ((1, 257), (64, 5), (65, 3)):
        dy, z, sc, sh, mean = TS.mask_case(n, 16, S, seed=n)
        y = np.maximum(TS.xhat(z, sc, sh), 0.0)
        TS.check_mask(z, sc, sh, y > 0)
        gam, beta = np.ones(16), np.zeros(16)
        got = emu_bn_affine_backward(dy, z, y, mean, sc, gam, beta, mutation)
        if mutation is None:
            TS.report(f"bn_backward at gamma = 1, n={n} S={S}", D.check_bn_affine_backward(dy, z, y, mean, sc, gam, *got))
        else:
            with pytest.raises(AssertionError):
                D.check_bn_affine_backward(dy, z, y, mean, sc, gam, *got)


@pytest.mark.parametrize("offset", [0.0, 1e3])
def test_point_layer_checks(offset):
    K, V, nv = 2, 420, 10
    inv, W, b, gam, beta = D.pnt_case(K, V, nv, offset, seed=3)
    mean, rstd, scale, shift = D.pnt_stats(inv, W, b, gam, beta)
    feat, arg = emu_pnt_forward(inv, W, b, scale, shift)
    assert feat[0, 0, 0] == 0 and arg[0, 0, 0] == 0
    D.check_pnt_forward(inv, W, b, scale, shift, feat, arg)
    with pytest.raises(AssertionError, match="first maximum"):
        D.check_pnt_forward(inv, W, b, scale, shift, *emu_pnt_forward(inv, W, b, scale, shift, "last_max"))
    dfeat = np.random.default_rng(0).normal(size=(K, 16, V))
    D.check_pnt_backward(inv, arg, feat, dfeat, W, b, mean, rstd, gam, emu_pnt_backward(inv, arg, feat, dfeat, W, b, mean, rstd, gam))
    if offset == 0:                                        # zero slots: R counted without them shifts m1, m2
        with pytest.raises(AssertionError):
            D.check_pnt_backward(inv, arg, feat, dfeat, W, b, mean, rstd, gam,
                                 emu_pnt_backward(inv, arg, feat, dfeat, W, b, mean, rstd, gam, "R_without_zero_slots"))


def test_pool_checks_reject_strict_eps_and_139_positions():
    K = 5
    x, w = D.pool_case(K, seed=1)
    f, desc, equi = emu_pool_forward(x, w)
    assert f[0, 3] == D.EPS and np.count_nonzero(f[0]) == 1
    D.check_pool_forward(x, w, f, desc, equi)
    with pytest.raises(AssertionError):
        D.check_pool_forward(x, w, *emu_pool_forward(x, w, "avg_139"))
    rng = np.random.default_rng(0)
    ddesc = rng.normal(size=(K, 32)).astype(np.float32)
    dequi = rng.normal(size=(K, 32, 7, 20)).astype(np.float32)
    for fv in (f, D.pool_f_cases(K)):
        D.check_pool_backward(x, w, fv, ddesc, dequi, *emu_pool_backward(x, w, fv, ddesc, dequi))
        with pytest.raises(AssertionError):
            D.check_pool_backward(x, w, fv, ddesc, dequi, *emu_pool_backward(x, w, fv, ddesc, dequi, "strict_gt"))


@pytest.mark.parametrize("mutation", ["dgrad_unflipped", "wrap_one_side", "wrap_elevation", "wgrad_drop_split"])
def test_cyl_check_rejects(mutation):
    rejected = 0
    for Din, ea in [(1, (0, 0)), (3, (6, 19))]:
        x5, w, b, dy = D.cyl_case(1, 4, 4, Din, seed=Din)
        x5[0, 1, Din - 1, ea[0], ea[1]] = np.nan
        D.check_cyl(x5, w, b, dy, *emu_cyl(x5, w, b, dy))
        try:
            D.check_cyl(x5, w, b, dy, *emu_cyl(x5, w, b, dy, mutation))
        except AssertionError:
            rejected += 1
    assert rejected == 2
