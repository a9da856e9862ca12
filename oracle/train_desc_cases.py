"""Edge inputs for the Desc training step's kernels (csrc/bx_train_desc.cu, one wrapper each in ops.py) and the float64
checks they are held to, shared by tests/test_train_desc_kernels_fp64_*.py and tests/test_train_step_fp64_gpu.py.

TEST INFRASTRUCTURE ONLY.  As in oracle/train_step_cases.py (whose gamma, ratio and layout helpers are used here): the
``check_*`` functions take the inputs and what an implementation returned (a kernel, or a float64 restatement of it on
the CPU), assert the bounds and return the largest ratio (err / bound) of each check.  Arrays are NumPy, channel-first
[n, C, S] unless named blocked.

Bounds.  u = 2^-53, gamma_k = k u / (1 - k u).  A sum whose every term passes through at most k roundings (a fused
multiply-add counts once) is within gamma_k sum |term| of the exact sum.  Reference sums are exact: ``math.fsum`` of the
terms, or ``dot2`` (products split exactly by Dekker's two-product, accumulated with error-free transformations:
within u |s| + gamma_n^2 sum |a b| of the exact dot product, Ogita, Rump and Oishi 2005), so a reference adds one
rounding (+1 in k) to the kernel's k.  Reduction depths follow the kernels' order:

* conv1x1, float64 (one thread per (sample, position), accumulator = bias, then Cin FMAs in channel order):
  gamma_{Cin+1} (|W|^T |x| + |b|); with ``out=`` the result is one more rounding of out + acc: gamma_{Cin+2} (... + |out|).
  A zero weight column with a zero bias writes exactly 0.
* cross_sums (grid Ca/4 Cb/4 x 64 splits of 256 threads): split s takes the contiguous rows [s per, (s + 1) per),
  per = ceil(R / 64), R = n S; thread t its rows t, t + 256, ... by FMA, so ceil(per / 256) roundings; 8 levels of the
  block tree; 64 in-order split additions: d = ceil(ceil(R/64) / 256) + 72, bound gamma_{d+1} |X|^T |D|.
* bn_backward (grid C/4 x 64 splits): split s takes samples s, s + 64, ...; a thread the positions p, p + 256, ...
  of them: d = ceil(n/64) ceil(S/256) + 72; sum dz x^ has the product's rounding more.  x^ = (z - mean) rstd is two
  roundings computed identically here.  The ReLU mask is the forward's: y > 0 for the output y of bn_apply.  dx =
  gamma rstd (dz - m1 - x^ m2) on the kernel's own m1, m2 (its sums / N): 2 gamma_3 (|dz| + |m1| + |x^ m2|) |gamma rstd|.
  The pool layer's affine BatchNorms and, with gamma = 1, the affine = False ones of CostNet and Cylindrical_Net.
* point layer: derived at check_pnt_forward / check_pnt_backward.
* pool layer: f = sum_p x w / 140 by a serial FMA chain (140 roundings, the division one more); the normalisations and
  their backward are at most 40 roundings deep on any term: 2 gamma_40 of the same expression on absolute values, the
  2 for the float64 reference's own evaluation.  ``F.normalize``'s clamp_min passes the gradient through the norm where
  |v| >= eps (torch's clamp_min backward), so at |v| = 1e-12 exactly the gradient is the projected one.
* cylindrical convolution: out and dx 2 gamma_{k+1} |W|^T |x| (k = Din 9 Cin, 9 Cout), dW (gamma_{ceil(R/64) + 65} +
  gamma_R) |x|^T |dy| (64 contiguous row ranges, DMMA within each, then the splits in order; the reference's autograd
  gamma_R).  NaN: the footprint of every output equals float64 F.conv3d on the padded input (circular azimuth, zero
  elevation), bit for bit.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from .train_step_cases import SPLITS, THREADS, U32, U64, from_blocked, gamma, ratio, to_blocked  # noqa: F401

EPS = 1e-12                     # F.normalize's eps
CYL_E, CYL_A, CYL_S = 7, 20, 140
NORM_DEPTH = 40                 # roundings on a term of an L2 normalisation or its backward (32-term sums + 8)

CONV1X1_SHAPES = [(32, 16), (16, 4), (16, 32), (4, 16), (4, 4), (4, 12), (4, 32), (12, 4), (12, 12), (12, 32), (32, 4),
                  (32, 12), (32, 32)]
CROSS_NS = [(1, 1), (1, 63), (1, 64), (1, 65), (1, 140), (512, 140)]        # (n, S): R = n S
CROSS_C = [(32, 16), (16, 4), (4, 4), (32, 32)]
BNA_N = (1, 2, 63, 64, 65, 512)


# ------------------------------------------------------------------------------------------------ exact sums
def _two_prod(a, b):
    p = a * b
    t = a * 134217729.0
    ah = t - (t - a)
    al = a - ah
    t = b * 134217729.0
    bh = t - (t - b)
    bl = b - bh
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def dot2(a, b, axis=0, extra=()):
    """sum over ``axis`` of a b (+ each array in ``extra``), accurate as if in twice the working precision, then rounded."""
    a, b = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64))
    a, b = np.moveaxis(a, axis, 0), np.moveaxis(b, axis, 0)
    if a.shape[0] > 4096 and int(np.prod(a.shape[1:])) < 300:     # few long sums: fsum of the exact product halves
        p, e = _two_prod(a, b)
        p, e = p.reshape(a.shape[0], -1), e.reshape(a.shape[0], -1)
        ex = [np.broadcast_to(np.asarray(v, np.float64), a.shape[1:]).reshape(-1) for v in extra]
        out = [math.fsum(p[:, i].tolist() + e[:, i].tolist() + [v[i] for v in ex]) for i in range(p.shape[1])]
        return np.array(out).reshape(a.shape[1:])
    s = np.zeros(a.shape[1:])
    c = np.zeros(a.shape[1:])

    def add(s, c, v):
        t = s + v
        z = t - s
        return t, c + ((s - (t - z)) + (v - z))

    for k in range(a.shape[0]):
        p, e = _two_prod(a[k], b[k])
        s, c = add(s, c, p)
        c = c + e
    for v in extra:
        s, c = add(s, c, np.broadcast_to(np.asarray(v, np.float64), s.shape))
    return s + c


def fsum_rows(a):
    return np.array([math.fsum(r) for r in np.asarray(a, np.float64).tolist()], np.float64)


# ------------------------------------------------------------------------------------------------ conv1x1 (float64)
def conv1x1_case(n, Cin, Cout, S, seed=0, live=None, live_in=None):
    """x [n, Cin, S], w [Cin, Cout], b [Cout], out0 [n, Cout, S] (nonzero, for ``out=``); ``live``: only the first
    ``live`` output channels have weights and bias (the attention's one channel padded to four, 16 -> 4); ``live_in``:
    only the first ``live_in`` input channels are nonzero, in x and in w's rows (its transpose 4 -> 16 in the backward,
    on dz2 whose channels 1-3 are zero)."""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(n, Cin, S)) * 10.0 ** rng.integers(-3, 4, (n, Cin, S))
    w = rng.normal(size=(Cin, Cout))
    b = rng.normal(size=Cout)
    out0 = rng.normal(size=(n, Cout, S)) * 1e2
    if live is not None:
        w[:, live:] = 0.0
        b[live:] = 0.0
        out0[:, live:] = 0.0
    if live_in is not None:
        x[:, live_in:] = 0.0
        w[live_in:] = 0.0
    return x, w, b, out0


def check_conv1x1(x, w, b, got, out0=None):
    Cin = x.shape[1]
    bb = np.zeros(w.shape[1]) if b is None else np.asarray(b, np.float64)
    extra = [bb[None, :, None]] + ([out0] if out0 is not None else [])
    ref = dot2(x[:, :, None, :], w[None, :, :, None], axis=1, extra=extra)
    ab = np.einsum("ncs,co->nos", np.abs(x), np.abs(w)) + np.abs(bb)[None, :, None]
    if out0 is None:
        bound = gamma(Cin + 1) * ab
    else:
        bound = gamma(Cin + 2) * (ab + np.abs(out0))
    got = np.asarray(got, np.float64)
    zero = (w == 0).all(0) & (bb == 0)
    if out0 is not None:
        zero = zero & (out0 == 0).all(axis=(0, 2))
    assert (got[:, zero] == 0).all(), "a zero-padded output channel is not exactly 0"
    return dict(conv1x1_f64=ratio(np.abs(got - ref), bound, "conv1x1 float64"))


# ------------------------------------------------------------------------------------------------ cross_sums
def cross_case(n, Ca, Cb, S, kind, seed=0):
    """X [n, Ca, S], D [n, Cb, S]: "offset" (mean 1e4, spread 1: the products cancel nowhere but carry 1e8), "const"
    (every channel one value), "random"."""
    rng = np.random.default_rng(seed)
    if kind == "offset":
        X = 1e4 + rng.uniform(-1, 1, (n, Ca, S))
        D = np.where(np.arange(Cb) % 2, -1e4, 1e4)[None, :, None] + rng.uniform(-1, 1, (n, Cb, S))
    elif kind == "const":
        X = np.broadcast_to((0.37 * np.arange(Ca) - 1.25)[None, :, None], (n, Ca, S)).copy()
        D = np.broadcast_to((0.11 * np.arange(Cb) + 0.013)[None, :, None], (n, Cb, S)).copy()
    else:
        X, D = rng.normal(size=(n, Ca, S)), rng.normal(size=(n, Cb, S))
    return X, D


def cross_depth(R):
    return math.ceil(math.ceil(R / SPLITS) / THREADS) + 8 + SPLITS


def check_cross_sums(X, D, got):
    n, Ca, S = X.shape
    Cb = D.shape[1]
    got = np.asarray(got, np.float64)
    assert got.shape == (Ca, Cb), got.shape
    Xr = X.transpose(1, 0, 2).reshape(Ca, -1)
    Dr = D.transpose(1, 0, 2).reshape(Cb, -1)
    ref = dot2(Xr.T[:, :, None], Dr.T[:, None, :], axis=0)
    ab = np.abs(Xr) @ np.abs(Dr).T
    return dict(cross_sums=ratio(np.abs(got - ref), gamma(cross_depth(n * S) + 1) * ab, "cross_sums"))


# ------------------------------------------------------------------------------------------------ bn_backward
def fwd_relu(z, scale, shift):
    """the forward's output bn_apply(z, scale, shift, relu): max(RN(z scale + shift), 0) (one fused multiply-add)."""
    from .train_step_cases import xhat
    return np.maximum(xhat(z, scale, shift), 0.0)


def bna_case(n, C, S, seed=0, pad=False):
    """The pool layer's BatchNorm + ReLU backward on edge inputs -> dy, z (channel-first), mean, rstd, gamma, beta [C]
    and the forward's scale, shift as patchnet.bn_scale_shift forms them (scale = gamma rstd, shift = beta - mean scale).
    Channel c % 4 (of the live ones): 0 -- z at the ReLU boundary: every z within 8 ulp of the root of
    z scale + shift = 0, where gamma ((z - mean) rstd) + beta and the folded form can round to opposite signs; 1 -- a dead
    channel (beta < 0 and every z below the mean); 2 -- a constant channel (z = mean, var = 0, rstd = 1 / sqrt(eps));
    3 -- generic.  ``pad``: the BN(1) route, channel 0 live (a boundary channel) and 1-3 all zero parameters.
    |dy| in [0.5, 1.5]: a mask flip moves dx by at least 0.5 |gamma rstd|."""
    rng = np.random.default_rng(seed)
    dy = rng.uniform(0.5, 1.5, (n, C, S)) * rng.choice([-1.0, 1.0], (n, C, S))
    z = np.zeros((n, C, S))
    mean, rstd, gam, beta = (np.zeros(C) for _ in range(4))
    live = 1 if pad else C
    for c in range(live):
        k = c % 4
        mean[c] = rng.uniform(-3, 3)
        var = 0.0 if k == 2 else rng.uniform(0.05, 4.0)
        rstd[c] = 1.0 / math.sqrt(var + 1e-5)
        gam[c] = rng.uniform(0.3, 2.0) * rng.choice([-1.0, 1.0]) if k != 1 else rng.uniform(0.3, 2.0)
        beta[c] = rng.uniform(-1.0, 1.0) if k != 1 else -rng.uniform(0.5, 1.0)
        if k == 0:
            sc = rstd[c] * gam[c]
            sh = -mean[c] * sc + beta[c]
            root = -sh / sc
            steps = rng.integers(-8, 9, (n, S))
            v = np.full((n, S), root)
            for s in range(1, 9):
                up, dn = np.nextafter(v, np.inf), np.nextafter(v, -np.inf)
                v = np.where(steps >= s, np.where(steps > 0, up, v), np.where(steps <= -s, dn, v))
            z[:, c] = v
        elif k == 1:
            z[:, c] = mean[c] - rng.uniform(1e-3, 2.0, (n, S)) * np.sign(gam[c])
        elif k == 2:
            z[:, c] = mean[c]
        else:
            z[:, c] = mean[c] + rng.normal(size=(n, S))
    scale = rstd * gam                       # patchnet.bn_scale_shift, in its order
    shift = -mean * scale + beta
    return dy, z, mean, rstd, gam, beta, scale, shift


def bna_depth(n, S):
    return math.ceil(n / SPLITS) * math.ceil(S / THREADS) + 8 + SPLITS


def mask_from_dx(dy, z, mean, rstd, gam, sums, dx):
    """The ReLU mask a bn_backward applied, read back from its dx (channels with gamma rstd != 0): the kernel's dz =
    dx / (gamma rstd) + m1 + x^ m2 is dy (kept) or 0 (masked), and |dy| >= 0.5 tells them apart."""
    n, C, S = z.shape
    N = n * S
    G = (gam * rstd)[None, :, None]
    xh = (z - mean[None, :, None]) * rstd[None, :, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        dz = dx / G + (sums[0] / N)[None, :, None] + xh * (sums[1] / N)[None, :, None]
    return np.abs(dz - dy) < 0.5 * np.abs(dy)


def check_bn_affine_backward(dy, z, y, mean, rstd, gam, dx, sums):
    """dx, sums [2, C] of bn_backward against the forward output y's mask."""
    n, C, S = z.shape
    N = n * S
    dx, sums = np.asarray(dx, np.float64), np.asarray(sums, np.float64)
    keep = np.asarray(y) > 0
    out = {}
    live = (gam * rstd) != 0
    got_mask = mask_from_dx(dy, z, mean, rstd, gam, sums, dx)
    bad = int((got_mask != keep)[:, live].sum())
    assert bad == 0, f"the backward's ReLU mask differs from the forward's y > 0 at {bad} elements"
    out["bna_mask_elems"] = 0.0
    xh = (z - mean[None, :, None]) * rstd[None, :, None]
    dz = np.where(keep, dy, 0.0)
    t0 = dz.transpose(1, 0, 2).reshape(C, -1)
    xr = xh.transpose(1, 0, 2).reshape(C, -1)
    d = bna_depth(n, S)
    out["bna_sum_dz"] = ratio(np.abs(sums[0] - fsum_rows(t0)), gamma(d + 1) * np.abs(t0).sum(1), "bn_affine sum dz")
    ref1 = dot2(t0.T, xr.T, axis=0)
    out["bna_sum_dzxh"] = ratio(np.abs(sums[1] - ref1), gamma(d + 2) * np.abs(t0 * xr).sum(1), "bn_affine sum dz x^")
    zero = ~keep.any(axis=(0, 2))
    assert (sums[:, zero] == 0).all(), "a channel the forward zeroed everywhere has a non-zero sum"
    G = (gam * rstd)[None, :, None]
    a1, a2 = (sums[0] / N)[None, :, None], (sums[1] / N)[None, :, None]
    ref = G * ((dz - a1) - xh * a2)
    bound = 2 * gamma(3) * (np.abs(dz) + np.abs(a1) + np.abs(xh * a2)) * np.abs(G)
    dead = zero | ~live
    assert (dx[:, dead] == 0).all(), "a dead or padding channel's dx is not exactly 0"
    out["bna_dx"] = ratio(np.abs(dx - ref), bound, "bn_affine dx")
    return out


# ------------------------------------------------------------------------------------------------ point layer
def pnt_stats(inv, W, b, gam, beta, eps=1e-5):
    """float64 batch statistics of y = W x + b over every sample of inv -> mean, rstd, scale, shift (bn_scale_shift's order)."""
    y = _pnt_y(inv, W, b).reshape(-1, 16)
    mean, var = y.mean(0), y.var(0)
    rstd = 1.0 / np.sqrt(var + eps)
    scale = rstd * gam
    return mean, rstd, scale, -mean * scale + beta


def pnt_case(K, V, nv, offset=0.0, seed=0):
    """inv [K, V, nv, 3] fp32 (the last 3 slots of every voxel zero when nv > 3 and there is no offset, as SPT's empty
    slots), W [16, 3], b, gamma, beta [16].  With at least 20 samples, voxel (0, 0)'s samples are moved along W[0] to 3
    standard deviations on the dead side of channel 0's ReLU (an all-dead voxel: feat 0, arg 0).  With ``offset`` the
    coordinates sit around offset (1, -1, 0.5), where the moment-derived dense sums cancel."""
    rng = np.random.default_rng(seed)
    inv = rng.normal(size=(K, V, nv, 3)) * 0.3 + offset * np.array([1.0, -1.0, 0.5])
    if nv > 3 and offset == 0:
        inv[:, :, nv - 3:] = 0.0
    W = rng.normal(size=(16, 3))
    b = rng.normal(size=16) * 0.1
    gam = rng.uniform(0.5, 1.5, 16)
    beta = rng.normal(size=16) * 0.2
    if K * V * nv >= 20:
        mean, rstd, _, _ = pnt_stats(inv.astype(np.float32), W, b, gam, beta)
        want = mean[0] - (3.0 + abs(beta[0]) / gam[0]) / rstd[0]
        yy = inv[0, 0] @ W[0] + b[0]
        inv[0, 0] += np.outer(want - yy, W[0] / np.dot(W[0], W[0]))
    return inv.astype(np.float32), W, b, gam, beta


def pnt_boundary_case(seed=0):
    """Samples at channel c's ReLU boundary: K = 2, V = 8, nv = 1, every voxel one sample; with the statistics of these
    samples, shift is replaced by -RN(y scale) of voxel (0, v) so that fma(y, scale, shift) is the product's rounding
    error: positive, negative or exactly 0.  -> inv, W, b, scale, shift, mean, rstd, gamma."""
    rng = np.random.default_rng(seed)
    inv = (rng.normal(size=(2, 8, 1, 3)) * 0.3).astype(np.float32)
    W = rng.normal(size=(16, 3))
    b = rng.normal(size=16) * 0.1
    gam = rng.uniform(0.5, 1.5, 16)
    beta = rng.normal(size=16) * 0.2
    mean, rstd, scale, shift = pnt_stats(inv, W, b, gam, beta)
    y = _pnt_y(inv, W, b)                                   # [2, 8, 1, 16]
    shift = -(y[0, 0, 0] * scale)                            # channel c: voxel (0, 0) sits on the boundary
    return inv, W, b, scale, shift, mean, rstd, gam


def _pnt_y(inv, W, b):
    x = np.asarray(inv, np.float32).astype(np.float64)
    return x @ W.T + b                                     # [K, V, nv, 16]


def check_pnt_forward(inv, W, b, scale, shift, feat, arg):
    """feat [K, 16, V] channel-first float64, arg [K, 16, V]: the first maximal sample of relu(y scale + shift).
    Per sample y is within gamma_4 (|W| |x| + |b|) in the kernel and in the reference, r = fma(y, scale, shift) within
    gamma_5 (|scale| (|W| |x| + |b|) + |shift|) each; ReLU and max are 1-Lipschitz, so a feature is within the largest
    per-sample bound (x 2, both sides) of its voxel."""
    x = np.asarray(inv, np.float32).astype(np.float64)
    y = _pnt_y(inv, W, b)
    r = np.maximum(y * scale + shift, 0.0)                  # [K, V, nv, 16]
    ref = r.max(2).transpose(0, 2, 1)                       # [K, 16, V]
    ref_arg = r.argmax(2).transpose(0, 2, 1)                # numpy's argmax: the first maximum
    ab = np.abs(scale) * (np.abs(x) @ np.abs(W).T + np.abs(b)) + np.abs(shift)
    bound = 2 * gamma(5) * ab.max(2).transpose(0, 2, 1)
    bad = int((np.asarray(arg) != ref_arg).sum())
    assert bad == 0, f"point layer: the selected sample differs from the first maximum at {bad} (patch, channel, voxel)"
    return dict(pnt_fwd=ratio(np.abs(np.asarray(feat, np.float64) - ref), bound, "point layer feat"))


def check_pnt_backward(inv, arg, feat, dfeat, W, b, mean, rstd, gam, out):
    """out [16, 6] = dW (3), db, dgamma, dbeta against the exact dense formula over all R = K V nv samples (zero slots
    included): dz_r = dfeat at the selected sample where the forward's feat > 0, m1 = S0 / R, m2 = S1 / R,
    dW = G (S_inv - m1 sum inv - m2 sum x^ inv), db = G (S0 - R m1 - m2 sum x^), dgamma = S1, dbeta = S0, G = gamma rstd.

    The kernel: S0..S4 over the selected samples, d_s = ceil(ceil(K V / 64) / 256) + 72 deep; the dense sums from the
    moments (each within gamma_{d_m} of its |terms|, d_m = ceil(R / 16384) + 72), sum x^ inv_j = rstd (W M_j + off mo_j),
    sum x^ = rstd (W mo + R off), off = b - mean, each with gamma_5 of its own evaluation; then the closing combination,
    gamma_4 of its |terms|.  x^_r itself (kernel and reference) within xi_r = rstd (gamma_4 (|W| |x_r| + |b|) + u |y_r -
    mean|) + u |x^_r|.  The moment errors times m2 rstd |off| are the cancellation term (~ rstd R |mean| u |m2|) that
    grows with an input offset.  The two sides' bounds are added, x 1.01 for the second-order terms."""
    K, V, nv, _ = inv.shape
    R = K * V * nv
    x = np.asarray(inv, np.float32).astype(np.float64)       # [K, V, nv, 3]
    y = _pnt_y(inv, W, b)                                     # [K, V, nv, 16]
    xh = (y - mean) * rstd
    ab_y = np.abs(x) @ np.abs(W).T + np.abs(b)
    xi = rstd * (gamma(4) * ab_y + U64 * np.abs(y - mean)) + U64 * np.abs(xh)
    feat = np.asarray(feat, np.float64)                      # [K, 16, V]
    sel = np.asarray(arg).astype(np.int64)                   # [K, 16, V]
    dfe = np.where(feat > 0, np.asarray(dfeat, np.float64), 0.0)
    dz = np.zeros((K, V, nv, 16))
    kk, cc, vv = np.meshgrid(np.arange(K), np.arange(16), np.arange(V), indexing="ij")
    dz[kk, vv, sel, cc] = dfe
    xr, dzr, xhr, xir = x.reshape(R, 3), dz.reshape(R, 16), xh.reshape(R, 16), xi.reshape(R, 16)
    S0 = np.array([math.fsum(dzr[:, c].tolist()) for c in range(16)])
    S1 = dot2(dzr, xhr, axis=0)
    Sj = dot2(dzr[:, :, None], xr[:, None, :], axis=0)       # [16, 3]
    sx = np.array([math.fsum(xr[:, j].tolist()) for j in range(3)])
    sxh = np.array([math.fsum(xhr[:, c].tolist()) for c in range(16)])
    sxi = dot2(xhr[:, :, None], xr[:, None, :], axis=0)      # [16, 3]
    G = gam * rstd
    m1, m2 = S0 / R, S1 / R
    ref_dW = G[:, None] * ((Sj - m1[:, None] * sx[None]) - m2[:, None] * sxi)
    ref_db = G * ((S0 - R * m1) - m2 * sxh)
    ad = np.abs(dzr)
    A0 = ad.sum(0)
    A1 = (ad * np.abs(xhr)).sum(0)
    Aj = ad.T @ np.abs(xr)                                    # [16, 3]
    # the kernel's sums, moments and dense sums
    ds = math.ceil(math.ceil(K * V / SPLITS) / THREADS) + 8 + SPLITS
    dm = math.ceil(R / (SPLITS * THREADS)) + 8 + SPLITS
    E_xi = (ad * xir).sum(0)                                  # x^'s own error in S1 (either side)
    eS0 = gamma(ds) * A0
    eS1 = gamma(ds + 1) * A1 + E_xi
    eSj = gamma(ds + 1) * Aj
    emo = gamma(dm) * np.abs(xr).sum(0)                       # [3]
    eM = gamma(dm) * (np.abs(xr).T @ np.abs(xr))              # [3, 3]
    mo = sx
    M = xr.T @ xr
    off = b - mean
    aW = np.abs(W)
    e_sxi = rstd[:, None] * (aW @ eM + np.abs(off)[:, None] * emo[None] + U64 * np.abs(off)[:, None] * np.abs(mo)[None]
                             + gamma(5) * (aW @ np.abs(M) + np.abs(off)[:, None] * np.abs(mo)[None])) + U64 * np.abs(sxi)
    e_sxh = rstd * (aW @ emo + R * U64 * np.abs(off) + gamma(5) * (aW @ np.abs(mo) + R * np.abs(off))) + U64 * np.abs(sxh)
    em1, em2 = eS0 / R + U64 * np.abs(m1), eS1 / R + U64 * np.abs(m2)
    aG = np.abs(G)
    k_dW = aG[:, None] * (eSj + np.abs(m1)[:, None] * emo[None] + em1[:, None] * np.abs(mo)[None] + np.abs(m2)[:, None] * e_sxi
                          + em2[:, None] * np.abs(sxi) + gamma(5) * (np.abs(Sj) + np.abs(m1[:, None] * mo[None]) + np.abs(m2[:, None] * sxi)))
    k_db = aG * (eS0 + R * em1 + np.abs(m2) * e_sxh + em2 * np.abs(sxh) + gamma(5) * (np.abs(S0) + R * np.abs(m1) + np.abs(m2 * sxh)))
    # the reference's own: x^ in sxi / sxh and the rounding of its combination
    r_dW = aG[:, None] * (np.abs(m2)[:, None] * (xir.T @ np.abs(xr)) + gamma(5) * (np.abs(Sj) + np.abs(m1[:, None] * mo[None])
                                                                               + np.abs(m2[:, None] * sxi)) + E_xi[:, None] / R * np.abs(sxi))
    r_db = aG * (np.abs(m2) * xir.sum(0) + E_xi / R * np.abs(sxh) + gamma(5) * (np.abs(S0) + R * np.abs(m1) + np.abs(m2 * sxh)))
    out = np.asarray(out, np.float64)
    res = {}
    res["pnt_dW"] = ratio(np.abs(out[:, :3] - ref_dW), 1.01 * (k_dW + r_dW), "point layer dW")
    res["pnt_db"] = ratio(np.abs(out[:, 3] - ref_db), 1.01 * (k_db + r_db), "point layer db")
    res["pnt_dgamma"] = ratio(np.abs(out[:, 4] - S1), 1.01 * (eS1 + E_xi + U64 * np.abs(S1)), "point layer dgamma")
    res["pnt_dbeta"] = ratio(np.abs(out[:, 5] - S0), eS0 + U64 * np.abs(S0), "point layer dbeta")
    return res


# ------------------------------------------------------------------------------------------------ pool layer
def _normalize_bwd(v, g):
    """torch's F.normalize(v, dim=0) and its backward on float64 columns v [C, P] -> (y, dv), via autograd."""
    vt = torch.from_numpy(np.ascontiguousarray(v, np.float64)).requires_grad_(True)
    yt = F.normalize(vt, dim=0, eps=EPS)
    yt.backward(torch.from_numpy(np.ascontiguousarray(g, np.float64)))
    return yt.detach().numpy(), vt.grad.numpy()


def _normalize_abs(v, g):
    """(|y| over the normalisation, |dv|'s absolute-value analog (|g| + |y| sum |y| |g|) / max(|v|, eps))."""
    n = np.sqrt((v * v).sum(0))
    den = np.maximum(n, EPS)
    ay = np.abs(v) / den
    return ay, (np.abs(g) + ay * (ay * np.abs(g)).sum(0)) / den


def pool_case(K, seed=0):
    """x [K, 32, 140], attention w [K, 140] >= 0, with the normalisation edges at patch 0 (if K allows): an equi position
    of norm exactly 1e-12 (one channel 1e-12), one ulp above and below it, one of norm 0; and an attention of 140 on a
    single position whose only nonzero channel is 1e-12, so f = [1e-12, 0, ...] (norm exactly 1e-12)."""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(K, 32, CYL_S))
    w = np.maximum(rng.normal(size=(K, CYL_S)), 0.0)
    x[0, :, 0:4] = 0.0
    x[0, 3, 0] = EPS
    x[0, 5, 1] = np.nextafter(EPS, np.inf)
    x[0, 7, 2] = np.nextafter(EPS, 0.0)
    w[0] = 0.0
    w[0, 0] = 140.0                       # f[0] = fl(fl(1e-12 140) / 140) = 1e-12 on channel 3, 0 elsewhere
    return x, w


def pool_f_cases(K, seed=0):
    """f [K, 32] rows for the backward: norm exactly 1e-12, one ulp above, one below, 0, then random."""
    rng = np.random.default_rng(seed + 1)
    f = rng.normal(size=(K, 32))
    edge = [EPS, np.nextafter(EPS, np.inf), np.nextafter(EPS, 0.0), 0.0]
    for i, v in enumerate(edge[:K]):
        f[i] = 0.0
        f[i, i] = v
    return f


def check_pool_forward(x, w, f, desc, equi):
    """f [K, 32] float64, desc [K, 32] and equi [K, 32, 140] fp32."""
    ref_f = dot2(x, w[:, None, :], axis=2) / CYL_S
    ab_f = (np.abs(x) * w[:, None, :]).sum(2) / CYL_S
    f = np.asarray(f, np.float64)
    out = dict(pool_f=ratio(np.abs(f - ref_f), gamma(CYL_S + 2) * ab_f, "pool f"))
    gd = NORM_DEPTH
    for name, v, got in (("pool_desc", f.T, np.asarray(desc, np.float64).T),
                         ("pool_equi", None, np.asarray(equi, np.float64).reshape(x.shape))):
        if v is None:
            ref = np.stack([F.normalize(torch.from_numpy(xk), dim=0, eps=EPS).numpy() for xk in x])
            ay = np.stack([_normalize_abs(xk, np.zeros_like(xk))[0] for xk in x])
        else:
            ref = F.normalize(torch.from_numpy(np.ascontiguousarray(v)), dim=0, eps=EPS).numpy()
            ay = _normalize_abs(v, np.zeros_like(v))[0]
        out[name] = ratio(np.abs(got - ref), U32 * np.abs(ref) + 2 * gamma(gd) * ay * (1 + U32), name)
    return out


def check_pool_backward(x, w, f, ddesc, dequi, dx, dw):
    """dx [K, 32, 140], dw [K, 140] (channel 0 of the blocked attention) from the kernel's f, torch's normalisation
    semantics (clamp_min: gradient through the norm where |v| >= eps)."""
    K = x.shape[0]
    dx, dw = np.asarray(dx, np.float64), np.asarray(dw, np.float64)
    ddesc, dequi = np.asarray(ddesc, np.float64), np.asarray(dequi, np.float64).reshape(K, 32, CYL_S)
    g = 2 * gamma(NORM_DEPTH)
    _, df = _normalize_bwd(f.T, ddesc.T)
    df = df.T                                                               # [K, 32]
    adf = _normalize_abs(f.T, ddesc.T)[1].T
    de = np.empty_like(x)
    ade = np.empty_like(x)
    for k in range(K):
        de[k] = _normalize_bwd(x[k], dequi[k])[1]
        ade[k] = _normalize_abs(x[k], dequi[k])[1]
    ref_dx = de + df[:, :, None] * w[:, None, :] / CYL_S
    e_df = g * adf
    b_dx = g * ade + e_df[:, :, None] * w[:, None, :] / CYL_S + 2 * gamma(3) * (np.abs(de) + np.abs(df[:, :, None] * w[:, None, :]) / CYL_S)
    ref_dw = (df[:, :, None] * x).sum(1) / CYL_S
    b_dw = ((e_df[:, :, None] * np.abs(x)).sum(1) + 2 * gamma(34) * (np.abs(df[:, :, None] * x)).sum(1)) / CYL_S
    return dict(pool_dx=ratio(np.abs(dx - ref_dx), b_dx, "pool dx"), pool_dw=ratio(np.abs(dw - ref_dw), b_dw, "pool dw"))


# ------------------------------------------------------------------------------------------------ cylindrical convolution
def pad_cyl(x):
    """[..., 7, 20] -> [..., 9, 22]: azimuth circular, elevation zero (utils/common.py's padding of patchnet.py)."""
    x = torch.cat([x[..., -1:], x, x[..., :1]], dim=-1)
    return F.pad(x, [0, 0, 1, 1])


def cyl_reference(x5, w, b, dy):
    """float64 F.conv3d on the padded input x5 [n, Cin, Din, 7, 20], w [Cout, Cin, Din, 3, 3] and its autograd backward
    from dy [n, Cout, 7, 20] -> (out, dx, dW) and the same on absolute values (for the bounds)."""
    def run(xa, wa, ba, dya):
        xt = torch.from_numpy(np.ascontiguousarray(xa)).requires_grad_(True)
        wt = torch.from_numpy(np.ascontiguousarray(wa)).requires_grad_(True)
        o = F.conv3d(pad_cyl(xt), wt, None if ba is None else torch.from_numpy(ba)).squeeze(2)
        o.backward(torch.from_numpy(np.ascontiguousarray(dya)))
        return o.detach().numpy(), xt.grad.numpy(), wt.grad.numpy()
    ref = run(x5, w, b, dy)
    ab = run(np.abs(np.nan_to_num(x5)), np.abs(w), np.abs(b), np.abs(np.nan_to_num(dy)))
    return ref, ab


def cyl_case(n, Cin, Cout, Din, seed=0):
    rng = np.random.default_rng(seed)
    x5 = rng.normal(size=(n, Cin, Din, CYL_E, CYL_A))
    w = rng.normal(size=(Cout, Cin, Din, 3, 3)) / math.sqrt(9 * Din * Cin)
    b = rng.normal(size=Cout)
    dy = rng.normal(size=(n, Cout, CYL_E, CYL_A))
    return x5, w, b, dy


def check_cyl(x5, w, b, dy, out, dx, dW):
    """out [n, Cout, 7, 20], dx like x5, dW like w: NaN footprints bit for bit, finite values within the bounds."""
    n, Cin, Din = x5.shape[:3]
    Cout = w.shape[0]
    (r_out, r_dx, r_dw), (a_out, a_dx, a_dw) = cyl_reference(x5, w, b, dy)
    res = {}
    R = n * CYL_S
    for name, got, ref, ab, g in (("cyl_out", out, r_out, a_out, 2 * gamma(Din * 9 * Cin + 1)),
                                  ("cyl_dx", dx, r_dx, a_dx, 2 * gamma(9 * Cout + 1)),
                                  ("cyl_dW", dW, r_dw, a_dw, gamma(math.ceil(R / SPLITS) + SPLITS + 1) + gamma(R))):
        got = np.asarray(got, np.float64)
        assert got.shape == ref.shape, (name, got.shape, ref.shape)
        gn, rn = np.isnan(got), np.isnan(ref)
        bad = int((gn != rn).sum())
        assert bad == 0, f"{name}: NaN footprint differs from float64 F.conv3d at {bad} elements"
        fin = ~rn
        res[name] = ratio(np.abs(got[fin] - ref[fin]), g * ab[fin], name)
    return res
