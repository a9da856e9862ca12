"""The Pose training step's checks (oracle/train_step_cases.py, where every bound is derived) without a GPU: each accepts
a float64 restatement of its kernel in csrc/bx_train_step.cu (the same split order, mask, index map and tap walk) and
rejects a subtly wrong one.  tests/test_train_step_fp64_gpu.py holds the kernels to the same checks.  The running-statistics
check also runs the module's own update rule, ``patchnet.bn_batch_stats``, which is plain torch."""
import math

import numpy as np
import pytest
import torch

from oracle import train_step_cases as C


# ------------------------------------------------------------------------------------------------ restatements
def emu_channel_sums(x, mutation=None):
    """channel-first float64 [n, C, S] -> [2, C]: per split (samples s = split mod 64) the partial sums, added in split order."""
    n, Cc, S = x.shape
    a = x.astype(np.float64)
    b = a * a
    out = np.zeros((2, Cc))
    for split in range(C.SPLITS):
        if mutation == "drop_split63" and split == 63:
            continue
        out[0] += a[split::C.SPLITS].sum(axis=(0, 2))
        out[1] += b[split::C.SPLITS].sum(axis=(0, 2))
    return out


def emu_moments3(v, mutation=None):
    a = v.astype(np.float64)
    x, y, z = a[:, 0], a[:, 1], a[:, 2]
    out = np.array([t.sum() for t in (x, y, z, x * x, x * y, x * z, y * y, y * z, z * z)])
    if mutation == "swap_xy_xz":
        out[[4, 5]] = out[[5, 4]]
    return out


def emu_softargmax(lg, g=None, mutation=None):
    e = np.exp(lg - lg.max(1, keepdims=True))
    k = np.arange(lg.shape[1])[None]
    se = e.sum(1, keepdims=True)
    r = (e * k).sum(1, keepdims=True) / se
    if g is None:
        return r[:, 0]
    return g[:, None] * (e / se) * (k if mutation == "no_minus_ind" else k - r)


def emu_costvol(s, t, mutation=None):
    M = s.shape[0]
    nn, l = np.arange(20)[:, None], np.arange(20)[None, :]
    idx = (l + nn) % 20 if mutation == "l_plus_nn" else (l - nn) % 20
    rows = slice(0, 5) if mutation == "rows_0_4" else slice(1, 6)
    s5, t5 = s[:, :, rows].astype(np.float64), t[:, :, rows].astype(np.float64)
    cv = s5[:, :, :, idx]                                 # [M, 32, k, nn, l]
    cv = cv.transpose(0, 1, 3, 2, 4) - t5[:, :, None]     # [M, 32, nn, k, l]
    return C.to_blocked(cv.reshape(M, 32, 2000))


def _taps(k):
    kd, kh, kw = k
    return [(a, b, c) for a in range(kd) for b in range(kh) for c in range(kw)]


def emu_conv_forward(x, w, b, mutation=None):
    n, Cin, D, H, W = x.shape
    Cout, _, kd, kh, kw = w.shape
    OD, OH, OW = D - kd + 1, H - kh + 1, W - kw + 1
    out = np.broadcast_to(b[None, :, None, None, None], (n, Cout, OD, OH, OW)).copy()
    for (a, bb, c) in _taps((kd, kh, kw)):
        ta, tb, tc = (kd - 1 - a, kh - 1 - bb, kw - 1 - c) if mutation == "flipped_tap" else (a, bb, c)
        out += np.einsum("ncdhw,oc->nodhw", x[:, :, ta:ta + OD, tb:tb + OH, tc:tc + OW], w[:, :, a, bb, c])
    return out


def emu_conv_dx(x, w, dy, mutation=None):
    """dx[ip] = sum_t W[t]^T dy[ip - t] (a convolution); the mutation correlates, dy[ip + t]."""
    n, Cin, D, H, W = x.shape
    Cout, _, kd, kh, kw = w.shape
    OD, OH, OW = dy.shape[2:]
    dx = np.zeros_like(x)
    for (a, b, c) in _taps((kd, kh, kw)):
        if mutation == "correlation":
            pad = np.zeros((n, Cout, D + kd, H + kh, W + kw))
            pad[:, :, :OD, :OH, :OW] = dy
            src = pad[:, :, a:a + D, b:b + H, c:c + W]
            dx += np.einsum("nodhw,oc->ncdhw", src, w[:, :, a, b, c])
        else:
            dx[:, :, a:a + OD, b:b + OH, c:c + OW] += np.einsum("nodhw,oc->ncdhw", dy, w[:, :, a, b, c])
    return dx


def emu_conv_dw(x, w, dy, mutation=None):
    """dW over 64 contiguous row ranges of ceil(R / 64) (sample, output position) rows, added in split order; the
    mutation loses the first row of every range."""
    n, Cin, D, H, W = x.shape
    Cout, _, kd, kh, kw = w.shape
    OD, OH, OW = dy.shape[2:]
    R = n * OD * OH * OW
    per = math.ceil(R / C.SPLITS)
    dyr = dy.transpose(0, 2, 3, 4, 1).reshape(R, Cout)
    dw = np.zeros_like(w)
    for (a, b, c) in _taps((kd, kh, kw)):
        xr = x[:, :, a:a + OD, b:b + OH, c:c + OW].transpose(0, 2, 3, 4, 1).reshape(R, Cin)
        for s in range(C.SPLITS):
            rb, re = per * s, min(R, per * s + per)
            if mutation == "drop_boundary_row":
                rb += 1
            if rb < re:
                dw[:, :, a, b, c] += dyr[rb:re].T @ xr[rb:re]
    return dw


def emu_running(rm0, rv0, nbt0, mean, var, N, momentum, mutation=None):
    m = momentum if momentum is not None else 1.0 / (nbt0 + 1)
    if mutation == "none_as_0.1" and momentum is None:
        m = 0.1
    corr = 1.0 if mutation == "biased_var" else N / (N - 1)
    rm0, rv0 = rm0.astype(np.float64), rv0.astype(np.float64)
    return (1 - m) * rm0 + m * mean, (1 - m) * rv0 + m * var * corr, nbt0 + 1


# ------------------------------------------------------------------------------------------------ checks on the restatements
def check_sums(mutation=None):
    acc = {}
    for n in C.SUM_N:
        for S in (1, 257, 2000) if n < 1000 else (4, 257):
            for kind in ("const", "positive", "offset"):
                for dt in (np.float32, np.float64):
                    x = C.sums_input(n, 4, S, kind, seed=n + S, dtype=dt)
                    C.merge(acc, C.check_channel_sums(x, emu_channel_sums(x, mutation=mutation)))
    return acc


def check_moments(mutation=None):
    acc = {}
    for R in (1, 255, 16385):
        for off in (0.0, 1e3):
            v = C.moments_input(R, off, seed=R)
            C.merge(acc, C.check_moments3(v, emu_moments3(v, mutation)))
    return acc


def check_sam(mutation=None):
    acc = {}
    for L in C.SAM_L:
        for kind in ("flat", "spread", "tied", "huge", "offset", "normal"):
            lg = C.sam_logits(129, L, kind, seed=L)
            g = np.random.default_rng(L).normal(size=129)
            g[::7] = 0.0
            C.merge(acc, C.check_softargmax(lg, emu_softargmax(lg)))
            C.merge(acc, C.check_softargmax_backward(lg, g, emu_softargmax(lg, g, mutation)))
    return acc


def check_cv(mutation=None):
    acc = {}
    for M, wide in ((1, False), (3, True)):
        s, t = C.costvol_maps(M, seed=M, wide=wide)
        C.merge(acc, C.check_costvol(s, t, emu_costvol(s, t, mutation)))
    return acc


def check_conv(mutation=None):
    acc = {}
    for (n, Cin, Cout, DHW, k) in [(2, 32, 20, (4, 1, 4), (3, 1, 3)), (65, 32, 20, (2, 1, 2), (2, 1, 2)),
                                   (3, 32, 8, (4, 3, 5), (2, 3, 1))]:
        x, w, b, dy = C.conv_case(n, Cin, Cout, DHW, k, seed=n)
        C.merge(acc, C.check_conv_forward(x, w, b, emu_conv_forward(x, w, b, mutation)))
        C.merge(acc, C.check_conv_dx(x, w, dy, emu_conv_dx(x, w, dy, mutation)))
        C.merge(acc, C.check_conv_dw(x, w, dy, emu_conv_dw(x, w, dy, mutation)))
    return acc


def check_running(mutation=None):
    acc = {}
    rng = np.random.default_rng(0)
    for N in (4, 12, 1000):
        for momentum in (0.1, None, 0.7):
            for nbt0 in (0, 3):
                rm0, rv0 = rng.normal(size=8).astype(np.float32), rng.uniform(0.5, 2, 8).astype(np.float32)
                mean, var = rng.normal(size=8), rng.uniform(0, 3, 8)
                rm, rv, nbt = emu_running(rm0, rv0, nbt0, mean, var, N, momentum, mutation)
                C.merge(acc, C.check_running_update(rm0, rv0, nbt0, mean, var, N, momentum,
                                                    np.float32(rm), np.float32(rv), nbt))
    return acc


def check_pnt(mutation=None):
    """patch_embedder.pnt_stats_from_moments (plain torch) on float64 moments of the samples."""
    from bufferx_b200.models.patch_embedder import pnt_stats_from_moments
    acc = {}
    rng = np.random.default_rng(4)
    W, b = rng.normal(size=(16, 3)) * 0.7, rng.normal(size=16) * 0.1
    for K, off in ((1, 0.0), (3, 1e3), (2, 10.0)):
        inv = C.pnt_inv_case(K, off, seed=K)
        mo = emu_moments3(inv.reshape(-1, 3), "swap_xy_xz" if mutation == "pnt_swap_xy_xz" else None) / (inv.size // 3)
        mean, var = pnt_stats_from_moments(torch.from_numpy(mo), torch.from_numpy(W), torch.from_numpy(b))
        C.merge(acc, C.check_pnt_stats(inv, W, b, mean.numpy(), var.numpy()))
    return acc


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("check", [check_sums, check_moments, check_sam, check_cv, check_conv, check_running, check_pnt],
                         ids=lambda f: f.__name__)
def test_restatement_passes(check):
    C.report(check.__name__, check())


MUTATIONS = [
    ("drop_split63", check_sums),
    ("no_minus_ind", check_sam),
    ("l_plus_nn", check_cv),
    ("rows_0_4", check_cv),
    ("flipped_tap", check_conv),
    ("correlation", check_conv),
    ("drop_boundary_row", check_conv),
    ("biased_var", check_running),
    ("none_as_0.1", check_running),
    ("swap_xy_xz", check_moments),
    ("pnt_swap_xy_xz", check_pnt),
]


@pytest.mark.parametrize("mutation,check", MUTATIONS, ids=[m for m, _ in MUTATIONS])
def test_mutation_is_caught(mutation, check):
    with pytest.raises(AssertionError):
        check(mutation)


def test_bn_batch_stats_follows_torch_running_update():
    """The module's update rule (patchnet.bn_batch_stats, plain torch) on a CPU BatchNorm, over three calls, for momentum
    0.1, None (the cumulative average) and N = 4 (N / (N - 1) = 4/3), against the running-update check."""
    import bufferx_b200.models.patchnet as pn
    rng = np.random.default_rng(1)
    for momentum, eps, N in ((0.1, 1e-5, 4), (None, 1e-3, 4), (None, 1e-5, 972), (0.3, 1e-5, 65)):
        bn = torch.nn.BatchNorm3d(8, momentum=momentum, eps=eps, affine=False)
        for _ in range(3):
            x = rng.normal(size=(N, 8)) * rng.uniform(0.1, 3, 8) + rng.normal(size=8)
            sums = torch.from_numpy(np.stack([x.sum(0), (x * x).sum(0)]))
            rm0, rv0, nbt0 = bn.running_mean.clone().numpy(), bn.running_var.clone().numpy(), int(bn.num_batches_tracked)
            mean, var = pn.bn_batch_stats(sums, N, bn)
            C.check_running_update(rm0, rv0, nbt0, mean.numpy(), var.numpy(), N, momentum,
                                   bn.running_mean.numpy(), bn.running_var.numpy(), int(bn.num_batches_tracked))


def test_running_bound_accumulates_over_updates():
    """Two cumulative-average updates from num_batches_tracked = 0 weigh the batch-statistic errors by 1 and 1/2."""
    bm, bv = C.running_bound([(1.0, 2.0), (4.0, 8.0)], None, 0, 4)
    assert (bm, bv) == pytest.approx((1.0 + 0.5 * 4.0, (2.0 + 0.5 * 8.0) * 4 / 3), rel=1e-15)
    bm, bv = C.running_bound([(1.0, 1.0)], 0.1, 7, 1001)
    assert (bm, bv) == pytest.approx((0.1, 0.1 * 1001 / 1000), rel=1e-15)


def test_fma64_is_correctly_rounded():
    """The exact-x^ helper against exact rational arithmetic, including products whose rounding error is the result."""
    from fractions import Fraction
    rng = np.random.default_rng(2)
    a, b = rng.normal(size=200) * 1e3, rng.normal(size=200)
    c = -(a * b)
    c[::3] = rng.normal(size=len(c[::3]))
    got = C.fma64(a, b, c)
    for ai, bi, ci, g in zip(a, b, c, got):
        assert g == float(Fraction(ai) * Fraction(bi) + Fraction(ci))
