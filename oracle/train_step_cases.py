"""Edge inputs for the Pose training step's kernels (csrc/bx_train_step.cu, one wrapper each in ops.py) and the float64
checks they are held to, shared by tests/test_train_step_fp64_*.py.

TEST INFRASTRUCTURE ONLY.  The ``check_*`` functions take the inputs and what an implementation returned (a kernel, or a
float64 restatement of it on the CPU), assert the bounds and return the largest ratio (err / bound) of each check
(``merge`` / ``report`` as in oracle/pose_cases.py).  Arrays are NumPy; blocked images are [n, C/4, S, 4].

Bounds.  u = 2^-53 (float64), 2^-24 (fp32); gamma_k = k u / (1 - k u).  A sum evaluated with at most k roundings on the
path of each term (a product, or a fused multiply-add, counts once) is within gamma_k sum |term| of the exact sum
(Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., sec. 3.1 and 4.2).  Reference sums are ``math.fsum``
over float64 terms: the correctly rounded exact sum.  The square or product of two fp32 values is exact in float64.

* channel_sums (grid C/4 x 64 splits of 256 threads): split s takes samples s, s + 64, ...; a thread adds the
  positions p, p + 256, ... of those samples, so one per-thread sum has ceil(n/64) ceil(S/256) terms; then 8 levels of
  the in-block tree and 64 in-order split additions: d = ceil(n/64) ceil(S/256) + 8 + 64.  With float64 inputs the
  product x^2 is rounded (or fused) in the kernel and rounded in the reference's terms: d + 1.
* moments3 (64 blocks x 256 threads, grid-strided): ceil(R / 16384) terms per thread, + 8 + 64, each of the 9 slots
  against its own fsum (products exact).
* bn_apply: y = fma(z, scale, shift), one rounding of the exact z scale + shift (bx_train_step.cu is built with FMA
  contraction).  fp32: |y - e| <= u32 |e|, e the exact value (z scale is exact in float64, e = RN64(z scale + shift) within
  u64 |e|): bound (u32 + 2 u64) |e|.  float64: the reference is RN(exact) (two-product + fsum) and the kernel one
  rounding of the same value: |y - ref| <= 2 u |ref| (1 + 2u).  With ReLU a value whose exact result is <= 0 is 0.
* ReLU mask: the forward's (bn_apply) is the sign of fma(z, scale, shift) bit for bit (the cases make z scale exact:
  power-of-two scales); the backward (bn_backward, held to oracle/train_desc_cases.check_bn_affine_backward with
  gamma = 1) reads it from the forward's output.
* conv1x1 (fp32 FMA chain, bias first): gamma32_{Cin+1} (|W|^T |x| + |b|), plus the float64 reference's own
  gamma64_{Cin+1} of the same.
* costvol: float64(s) - float64(t) is one IEEE subtraction on both sides: equal bits.
* softargmax (float64, one thread per row): with delta_k = l_k - max, the subtraction is within u |delta_k| and exp
  within 1 ulp (2u relative), so e_k carries eps_k = expm1(u |delta_k|) + 2u exp(u |delta_k|); se and sk = sum e_k k
  carry gamma_L more.  ind = sk / se: |d ind| <= (|d sk| + ind |d se|) / (se - |d se|) + u ind.  Backward
  dl_k = g p_k (k - ind): |d dl_k| <= |g| p_k (|k - ind| (eps_k + eps_se + 4u) + |d ind|), eps_se = sum e_k eps_k / se
  + gamma_L; every e_k and dl_k may also carry an absolute error of the subnormal spacing (exp underflowing).
  Reference: the same formula in extended precision (np.longdouble, u <= 2^-64: its own error is below 2^-11 of these
  bounds), bounds x 1.01 for the second-order terms.
* point layer statistics from moments: derived at check_pnt_stats.
* conv_forward: each output is T Cin products + bias, summed by FMAs (kernel) and by an unknown order (F.conv3d in
  float64): 2 gamma_{T Cin + 1} (|W|^T |x| + |b|), the contraction taken by the same convolution on absolute values.
* conv_backward: dW[t][ci][co] sums R = n S_out products in 64 contiguous row ranges of ceil(R/64) rows, 4 row groups
  added in order, then the 64 splits: d = ceil(R/64) + 3 + 64; the float64 reference (autograd) adds gamma_R: bound
  (gamma_d + gamma_R) |x|^T |dy|.  dx sums at most T Cout products: 2 gamma_{T Cout + 1} |W| * |dy| (transposed).
* running statistics: one update is r <- (1 - m) r + m v (N / (N - 1) for the variance), m = momentum or, with
  momentum None, 1 / num_batches_tracked after the increment.  An error b in the batch statistic moves r by at most
  m b, and (1 - m) <= 1 carries earlier errors unamplified, so after k updates the bound is sum_k m_k b_k (x N/(N-1)).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from .pose_cases import merge  # noqa: F401  (re-exported for the tests)

U64 = 2.0 ** -53
U32 = 2.0 ** -24
SPLITS = 64                    # BX_TS_SPLITS
THREADS = 256                  # TS_THREADS
TINY = 2.0 ** -1072            # the absolute error of a sum of exps in (or rounded into) the subnormal range, with room

SUM_N = (1, 63, 64, 65, 1000)
SUM_S = (1, 4, 255, 256, 257, 972, 2000)
MOM_R = (1, 255, 256, 16383, 16384, 16385, 512 * 4200)
SAM_L = (1, 2, 19, 20, 21, 64)
SAM_M = (1, 127, 128, 129, 4097)
COSTVOL_M = (1, 2, 3, 65, 1000)

# CostNet's ten layers: (Cin, Cout, (D, H, W) of the input, (kd, kh, kw))
COSTNET_GEOMS = [(32, 32, (20, 5, 20), (3, 3, 3)), (32, 64, (18, 3, 18), (3, 3, 3)), (64, 64, (16, 1, 16), (3, 1, 3)),
                 (64, 128, (14, 1, 14), (3, 1, 3)), (128, 128, (12, 1, 12), (3, 1, 3)), (128, 64, (10, 1, 10), (3, 1, 3)),
                 (64, 64, (8, 1, 8), (3, 1, 3)), (64, 32, (6, 1, 6), (3, 1, 3)), (32, 32, (4, 1, 4), (3, 1, 3)),
                 (32, 20, (2, 1, 2), (2, 1, 2))]
# synthetic shapes: (n, Cin, Cout, (D, H, W), (kd, kh, kw)); kernel == extent, 1x1x1 kernels, n S_out in {1, 63, 64, 65}
SYNTH_GEOMS = [(1, 32, 4, (3, 2, 4), (3, 2, 4)), (63, 96, 20, (2, 3, 2), (2, 3, 2)), (64, 160, 36, (1, 1, 1), (1, 1, 1)),
               (65, 32, 100, (2, 1, 3), (2, 1, 3)), (1, 96, 132, (3, 3, 7), (1, 1, 1)), (1, 160, 4, (1, 1, 64), (1, 1, 1)),
               (1, 32, 132, (7, 1, 15), (3, 1, 3)), (3, 96, 20, (4, 3, 5), (2, 3, 1)), (63, 32, 36, (1, 2, 2), (1, 1, 2))]


def gamma(k, u=U64):
    assert k * u < 1
    return k * u / (1.0 - k * u)


def report(name, out):
    ratios = {k: v for k, v in out.items() if isinstance(v, float)}
    print(f"\n[train-step-fp64] {name}: " + ", ".join(f"{k} {v:.3g}" for k, v in ratios.items()))


def ratio(err, bound, what):
    """max err / bound (bound 0: err must be 0); asserts <= 1 and returns it."""
    err, bound = np.asarray(err), np.asarray(bound)
    if err.dtype != np.longdouble:
        err, bound = err.astype(np.float64), bound.astype(np.float64)
    assert not np.isnan(err).any(), f"{what}: NaN"
    r = np.divide(err, bound, out=np.where(err > 0, np.inf, 0.0).astype(err.dtype), where=bound > 0)
    m = float(r.max()) if r.size else 0.0
    assert m <= 1.0, f"{what}: err {m:.3g} x bound"
    return m


def fsum_rows(a):
    """exact (correctly rounded) sums of the rows of a float64 array [R, K]."""
    return np.array([math.fsum(r) for r in np.asarray(a, np.float64).tolist()], np.float64)


def to_blocked(x):
    """channel-first [n, C, S] -> blocked [n, C/4, S, 4]."""
    n, C, S = x.shape
    return np.ascontiguousarray(x.reshape(n, C // 4, 4, S).transpose(0, 1, 3, 2))


def from_blocked(x):
    n, G, S, _ = x.shape
    return np.ascontiguousarray(x.transpose(0, 1, 3, 2).reshape(n, 4 * G, S))


def _split(a):
    t = a * 134217729.0
    hi = t - (t - a)
    return hi, a - hi


def fma64(a, b, c):
    """correctly rounded a b + c elementwise in float64 (Dekker's two-product, then fsum where the product is inexact)."""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(c, np.float64))
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    out = p + c
    idx = np.nonzero(e)
    if idx[0].size:
        out[idx] = [math.fsum(t) for t in zip(p[idx].tolist(), e[idx].tolist(), c[idx].tolist())]
    return out


# ------------------------------------------------------------------------------------------------ channel sums
def sums_input(n, C, S, kind, seed=0, dtype=np.float32):
    """channel-first [n, C, S]: "const" (every channel one value), "positive" (all > 0, so a dropped split lowers every
    sum), "offset" (means 1e4 x the spread, alternating sign)."""
    rng = np.random.default_rng(seed)
    c = np.arange(C)
    if kind == "const":
        x = np.broadcast_to((0.37 * c - 1.25 + 0.013)[None, :, None], (n, C, S))
    elif kind == "positive":
        x = rng.uniform(0.5, 1.5, (n, C, S)) * (1.0 + c)[None, :, None]
    else:
        x = np.where(c % 2, -1e4, 1e4)[None, :, None] + rng.uniform(-1, 1, (n, C, S))
    return np.ascontiguousarray(x.astype(dtype))


def sums_depth(n, S, f64):
    return math.ceil(n / SPLITS) * math.ceil(S / THREADS) + 8 + SPLITS + (1 if f64 else 0)


def check_channel_sums(x, got):
    """x channel-first [n, C, S] (fp32 or float64), got [2, C]: (sum x, sum x^2)."""
    n, C, S = x.shape
    x64 = x.astype(np.float64).transpose(1, 0, 2).reshape(C, -1)
    g = gamma(sums_depth(n, S, x.dtype == np.float64))
    got = np.asarray(got, np.float64)
    sq = x64 * x64
    out = {}
    out["sum"] = ratio(np.abs(got[0] - fsum_rows(x64)), g * np.abs(x64).sum(1), "sum x")
    out["sumsq"] = ratio(np.abs(got[1] - fsum_rows(sq)), g * sq.sum(1), "sum x^2")
    return out


def mask_case(n, C, S, seed=0):
    """The edge inputs of a BatchNorm with affine = False, channel-first float64 -> (dy, z, scale [C], shift [C], mean [C]):
    the forward is x^ = fma(z, scale, shift) with scale = rstd and shift = -RN(mean scale), as patchnet.bn_scale_shift
    forms them.  Channel c % 4 (mean z0):
    0 -- power-of-two scale, shift = -z0 scale (exact), about a third of the elements at z0 (x^ exactly 0) and at z0 +-1 ulp;
    1 -- as 0 but every z < z0 (a dead channel: dz = 0, m1 = m2 = 0); 2 -- constant z = z0 with the scale of var = 0,
    1 / sqrt(1e-5) (the forward's x^ the product's rounding error, (z - mean) rstd exactly 0); 3 -- a generic channel.
    |dy| in [0.5, 1.5]: a mask flip moves dx by at least 0.5 |scale|."""
    rng = np.random.default_rng(seed)
    dy = rng.uniform(0.5, 1.5, (n, C, S)) * rng.choice([-1.0, 1.0], (n, C, S))
    z = np.empty((n, C, S))
    scale, mean = np.empty(C), np.empty(C)
    for c in range(C):
        k = c % 4
        z0 = mean[c] = rng.uniform(-3, 3)
        if k in (0, 1):
            scale[c] = 2.0 ** int(rng.integers(-3, 4))
            v = z0 + rng.uniform(-2, 2, (n, S)) if k == 0 else z0 - rng.uniform(1e-3, 2, (n, S))
            if k == 0:
                pick = rng.integers(0, 6, (n, S))
                v = np.where(pick == 0, z0, np.where(pick == 1, np.nextafter(z0, np.inf), np.where(pick == 2, np.nextafter(z0, -np.inf), v)))
            z[:, c] = v
        elif k == 2:
            scale[c] = 1.0 / math.sqrt(1e-5)
            z[:, c] = z0
        else:
            scale[c] = rng.uniform(0.2, 3)
            z[:, c] = z0 + rng.normal(size=(n, S))
    return dy, z, scale, -(mean * scale), mean


def xhat(z, scale, shift):
    """x^ = RN(z scale + shift), channel-first [n, C, S] (the kernels' fused multiply-add)."""
    return fma64(z, scale[None, :, None], shift[None, :, None])


def check_mask(z, scale, shift, mask, xh=None):
    """A ReLU mask (bool, channel-first) against the exact sign of x^: equal bit for bit."""
    ref = (xhat(z, scale, shift) if xh is None else xh) > 0
    bad = int((np.asarray(mask, bool) != ref).sum())
    assert bad == 0, f"ReLU mask differs from x^ > 0 at {bad} elements"
    return dict(mask_elems=float(0))


# ------------------------------------------------------------------------------------------------ bn_apply
def apply_case(n, C, S, seed=0, dtype=np.float32):
    """channel-first z and per-channel (scale, shift) with shift ~ -mean scale (cancellation), each channel's shift
    10 apart from its neighbours' so a wrong channel index shows."""
    rng = np.random.default_rng(seed)
    mean = rng.uniform(-5, 5, C)
    z = (mean[None, :, None] + rng.normal(size=(n, C, S))).astype(dtype)
    scale = rng.uniform(0.3, 3, C).astype(dtype)
    shift = (-mean * scale + 10.0 * (np.arange(C) - C / 2) * rng.uniform(0, 1, C) * (np.arange(C) % 2)).astype(dtype)
    return z, scale, shift


def check_bn_apply(z, scale, shift, relu, got):
    got = np.asarray(got, np.float64)
    if z.dtype == np.float32:
        e = z.astype(np.float64) * scale.astype(np.float64)[None, :, None] + shift.astype(np.float64)[None, :, None]
        bound = (U32 + 2 * U64) * np.abs(e)
    else:
        e = xhat(z, scale, shift)
        bound = 2 * U64 * (1 + 2 * U64) * np.abs(e)
    if relu:
        bound = np.where(e > 0, bound, 0.0)
        e = np.maximum(e, 0.0)
    return dict(bn_apply=ratio(np.abs(got - e), bound, "bn_apply"))


# ------------------------------------------------------------------------------------------------ moments3
def moments_input(R, offset, seed=0):
    """[R, 3] fp32: axes of different offsets and spreads, so the nine slots differ."""
    rng = np.random.default_rng(seed)
    v = rng.uniform(-1, 1, (R, 3)) * np.array([1.0, 0.5, 2.0]) + offset * np.array([1.0, -1.0, 0.5])
    return np.ascontiguousarray(v.astype(np.float32))


MOMENT_SLOTS = ["x", "y", "z", "xx", "xy", "xz", "yy", "yz", "zz"]


def check_moments3(v, got):
    R = v.shape[0]
    a = v.astype(np.float64)
    x, y, z = a[:, 0], a[:, 1], a[:, 2]
    terms = [x, y, z, x * x, x * y, x * z, y * y, y * z, z * z]
    g = gamma(math.ceil(R / (SPLITS * THREADS)) + 8 + SPLITS)
    got = np.asarray(got, np.float64)
    out = {}
    for i, (name, t) in enumerate(zip(MOMENT_SLOTS, terms)):
        out[f"m_{name}"] = ratio(abs(got[i] - math.fsum(t.tolist())), g * np.abs(t).sum(), f"moments3 slot {name}")
    return out


def check_pnt_stats(inv, W, b, mean, var, depth=None):
    """The point layer's batch statistics from moments (patch_embedder.pnt_stats_from_moments on moments3 / R) against a
    float64 BatchNorm over the explicit outputs y = W x + b of the R samples ``inv`` [..., 3] (fp32), W [16, 3], b [16].

    The route: S_i = sum x_i and S_ij = sum x_i x_j within gamma_d of the sums of |terms| (A_i, A_ij; d = ``depth``, the
    moments3 depth ceil(R/16384) + 72 by default), then / R: e_i = gamma_{d+1} A_i / R, e_ij = gamma_{d+1} A_ij / R.
    cov_ij = E[x_i x_j] - E[x_i] E[x_j] within e_ij + |Ex_i| e_j + |Ex_j| e_i + e_i e_j + gamma_2 (|Exx_ij| + |Ex_i Ex_j|).
    mean_c = W_c Ex + b_c (3 products, 3 additions) within sum_i |W_ci| e_i + gamma_4 (sum_i |W_ci| |Ex_i| + |b_c|);
    var_c = sum_j (sum_i W_ci cov_ij) W_cj within sum_ij |W_ci| |W_cj| dcov_ij + gamma_6 sum_ij |W_ci| |cov_ij| |W_cj|
    (the clamp at 0 only moves a value toward the non-negative truth).
    The reference: y_r in float64 within eta_r = gamma_4 (sum_i |W_ci| |x_ri| + |b_c|); mean = fsum(y) / R within
    mean |eta| + 2u |mean|; var = fsum(d_r^2) / R with d_r = y_r - mean, each d_r within err_r = eta_r + dmean + u |d_r|:
    within mean_r(2 |d_r| err_r + err_r^2 + u d_r^2) + 2u var.  Both bounds are evaluated at the float64 values, their sum
    x 1.01 for the second-order terms.  With coordinates offset by 1e3, E[xx] ~ 1e6 cancels to a covariance of ~1, and
    e_ij is what the variance bound is made of."""
    x = np.asarray(inv, np.float32).reshape(-1, 3).astype(np.float64)
    R = x.shape[0]
    W, b = np.asarray(W, np.float64), np.asarray(b, np.float64)
    d = math.ceil(R / (SPLITS * THREADS)) + 8 + SPLITS if depth is None else depth
    g = gamma(d + 1)
    A = np.abs(x).sum(0)
    Aij = np.abs(x).T @ np.abs(x)
    Ex = np.array([math.fsum(x[:, i].tolist()) for i in range(3)]) / R
    Exx = np.array([[math.fsum((x[:, i] * x[:, j]).tolist()) for j in range(3)] for i in range(3)]) / R
    cov = Exx - np.outer(Ex, Ex)
    e, eij = g * A / R, g * Aij / R
    aE = np.abs(Ex)
    dcov = eij + np.outer(aE, e) + np.outer(e, aE) + np.outer(e, e) + gamma(2) * (np.abs(Exx) + np.outer(aE, aE))
    aW = np.abs(W)
    b_mean = aW @ e + gamma(4) * (aW @ aE + np.abs(b))
    b_var = np.einsum("ci,ij,cj->c", aW, dcov, aW) + gamma(6) * np.einsum("ci,ij,cj->c", aW, np.abs(cov), aW)
    y = x @ W.T + b
    eta = gamma(4) * (np.abs(x) @ aW.T + np.abs(b))
    m_ref = np.array([math.fsum(y[:, c].tolist()) for c in range(y.shape[1])]) / R
    dm = eta.mean(0) + 2 * U64 * np.abs(m_ref)
    dd = y - m_ref
    v_ref = np.array([math.fsum((dd[:, c] ** 2).tolist()) for c in range(y.shape[1])]) / R
    er = eta + dm + U64 * np.abs(dd)
    dv = (2 * np.abs(dd) * er + er * er + U64 * dd * dd).mean(0) + 2 * U64 * v_ref
    mean, var = np.asarray(mean, np.float64), np.asarray(var, np.float64)
    return dict(pnt_mean=ratio(np.abs(mean - m_ref), 1.01 * (b_mean + dm), "point-layer batch mean"),
                pnt_var=ratio(np.abs(var - v_ref), 1.01 * (b_var + dv), "point-layer batch variance"))


def pnt_inv_case(K, offset, seed=0, nv=10):
    """De-rotated point-layer inputs [K, 420, nv, 3] fp32: points in a unit ball around ``offset`` (1, -1, 0.5); without an
    offset a quarter of the slots are zero, as the SPT's empty voxel slots are (with one, none: so the covariance cancels)."""
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(K, 420, nv, 3)) * 0.3 + offset * np.array([1.0, -1.0, 0.5])
    if offset == 0:
        v[rng.random((K, 420, nv)) < 0.25] = 0.0
    return np.ascontiguousarray(v.astype(np.float32))


# ------------------------------------------------------------------------------------------------ conv1x1
def check_conv1x1(x, w, b, got):
    """x channel-first fp32 [n, Cin, S], w [Cin, Cout4], b [Cout4] -> got channel-first [n, Cout4, S]."""
    x64, w64, b64 = x.astype(np.float64), w.astype(np.float64), b.astype(np.float64)
    ref = np.einsum("ncs,co->nos", x64, w64) + b64[None, :, None]
    ab = np.einsum("ncs,co->nos", np.abs(x64), np.abs(w64)) + np.abs(b64)[None, :, None]
    k = x.shape[1] + 1
    got = np.asarray(got, np.float64)
    zero = (w == 0).all(0) & (b == 0)
    assert (got[:, zero] == 0).all(), "a zero-padded output channel is not exactly 0"
    return dict(conv1x1=ratio(np.abs(got - ref), (gamma(k, U32) + gamma(k)) * ab, "conv1x1"))


# ------------------------------------------------------------------------------------------------ cost volume
def costvol_maps(M, seed=0, wide=False):
    """fp32 [M, 32, 7, 20] pairs; ``wide``: magnitudes 1e30 and 1e-30 mixed (the float64 difference rounds); elevation
    rows 0 and 6 NaN (never read)."""
    rng = np.random.default_rng(seed)
    s, t = rng.normal(size=(2, M, 32, 7, 20))
    if wide:
        s *= np.where(rng.random(s.shape) < 0.5, 1e30, 1e-30)
        t *= np.where(rng.random(t.shape) < 0.5, 1e30, 1e-30)
    s, t = s.astype(np.float32), t.astype(np.float32)
    s[:, :, [0, 6]] = np.nan
    t[:, :, [0, 6]] = np.nan
    return s, t


def costvol_ref(s, t):
    """the oracle's cost_volume of rows 1..5 in float64, blocked [M, 8, 2000, 4]."""
    from .train_step import cost_volume
    cv = cost_volume(torch.from_numpy(s[:, :, 1:6]).double(), torch.from_numpy(t[:, :, 1:6]).double()).numpy()
    M = s.shape[0]
    return to_blocked(cv.reshape(M, 32, 2000))


def check_costvol(s, t, got):
    ref = costvol_ref(s, t)
    got = np.asarray(got, np.float64)
    assert got.shape == ref.shape
    bad = int((got.view(np.int64) != ref.view(np.int64)).sum())
    assert bad == 0, f"cost volume differs from float64(s) - float64(t) at {bad} elements"
    return dict(costvol_bits=0.0)


# ------------------------------------------------------------------------------------------------ soft arg-max
def sam_logits(M, L, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "flat":
        return np.full((M, L), 0.75)
    if kind == "spread":                 # 1e3: exp underflows, ind is (nearly) an exact integer
        return rng.uniform(-1, 1, (M, L)) * 1e3
    if kind == "tied":                   # maxima at 0 and L - 1
        x = rng.uniform(-3, 0, (M, L))
        x[:, 0] = x[:, L - 1] = 1.0
        return x
    if kind == "huge":                   # 1e300 offsets: any two distinct logits differ by >= ulp(1e300) ~ 1.5e284, so
        return 1e300 * (1.0 + rng.integers(0, 4, (M, L)) * 2.0 ** -52)   # only the tied maxima survive the max subtraction
    if kind == "offset":                 # 1e12 offset, O(1) spread: the logits and their differences carry ulp(1e12)
        return 1e12 + rng.normal(size=(M, L)) * 2.0
    return rng.normal(size=(M, L)) * 3.0


def _sam_terms(logits):
    lg = np.asarray(logits, np.float64)
    M, L = lg.shape
    ld = lg.astype(np.longdouble)
    mx = ld.max(1, keepdims=True)
    e = np.exp(ld - mx)
    k = np.arange(L, dtype=np.longdouble)[None]
    se, sk = e.sum(1, keepdims=True), (e * k).sum(1, keepdims=True)
    ind = sk / se
    dlt = np.abs(lg - lg.max(1, keepdims=True))
    e64 = e.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        eps = np.expm1(U64 * dlt) + 2 * U64 * np.exp(U64 * dlt)
        ek = np.where(e64 > 0, e64 * eps, 0.0) + TINY
    gL = gamma(L + 1)
    dse = ek.sum(1, keepdims=True) + gL * e64.sum(1, keepdims=True)
    dsk = (ek * np.arange(L)[None]).sum(1, keepdims=True) + gL * (e64 * np.arange(L)[None]).sum(1, keepdims=True)
    se64, ind64 = se.astype(np.float64), ind.astype(np.float64)
    dind = (dsk + ind64 * dse) / (se64 - dse) + U64 * ind64
    return dict(e=e, se=se, ind=ind, eps=eps, eps_se=dse / se64, dind=dind, L=L)


def check_softargmax(logits, ind):
    """forward: ind [M] within 1.01 x the derived bound of the extended-precision formula."""
    assert np.finfo(np.longdouble).eps <= 2.0 ** -63, "the soft arg-max reference needs an extended long double"
    t = _sam_terms(logits)
    ref, b = t["ind"][:, 0].astype(np.float64), 1.01 * t["dind"][:, 0]
    return dict(sam_fwd=ratio(np.abs(np.asarray(ind, np.float64) - ref), b, "softargmax ind"))


def check_softargmax_backward(logits, g, dl):
    """backward: dlogits [M, L] within 1.01 x the derived bound; sum_k dl_k = 0 within the sum of the bounds; g = 0 rows 0.
    Evaluated in extended precision, where the bounds of subnormal results do not underflow."""
    t = _sam_terms(logits)
    L = t["L"]
    p = t["e"] / t["se"]
    k = np.arange(L, dtype=np.longdouble)[None]
    g = np.asarray(g, np.float64).astype(np.longdouble)
    ref = g[:, None] * p * (k - t["ind"])
    kr = np.abs(k - t["ind"])
    with np.errstate(invalid="ignore", over="ignore"):
        b = 1.01 * np.abs(g)[:, None] * p * (kr * (t["eps"] + t["eps_se"] + 4 * U64) + t["dind"])
    b = np.where(p > 0, b, 0.0) + 2 * (np.abs(g)[:, None] + 1) * (kr + 1) * np.longdouble(2.0 ** -1074)
    dl64 = np.asarray(dl, np.float64)
    dl = dl64.astype(np.longdouble)
    out = dict(sam_bwd=ratio(np.abs(dl - ref), b, "softargmax dlogits"))
    out["sam_bwd_sum"] = ratio(np.abs(fsum_rows(dl64)), b.sum(1), "softargmax sum_k dlogits")
    assert (dl64[np.asarray(g) == 0] == 0).all(), "g = 0 gives a non-zero dlogit"
    return out


# ------------------------------------------------------------------------------------------------ convolutions
def conv_case(n, Cin, Cout, DHW, k, seed=0):
    """float64 x [n, Cin, D, H, W], W [Cout, Cin, kd, kh, kw] (random, so asymmetric), b [Cout], dy like the output."""
    rng = np.random.default_rng(seed)
    D, H, W = DHW
    kd, kh, kw = k
    x = rng.normal(size=(n, Cin, D, H, W))
    w = rng.normal(size=(Cout, Cin, kd, kh, kw)) / math.sqrt(Cin * kd * kh * kw)
    b = rng.normal(size=Cout)
    dy = rng.normal(size=(n, Cout, D - kd + 1, H - kh + 1, W - kw + 1))
    return x, w, b, dy


def wt_of(w):
    """[Cout, Cin, kd, kh, kw] -> the kernels' Wt [T, Cin, Cout]."""
    return np.ascontiguousarray(w.reshape(w.shape[0], w.shape[1], -1).transpose(2, 1, 0))


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float64))


def check_conv_forward(x, w, b, got):
    """got [n, Cout, OD, OH, OW] against F.conv3d in float64: 2 gamma_{T Cin + 1} (|W|^T |x| + |b|)."""
    ref = F.conv3d(_t(x), _t(w), _t(b)).numpy()
    ab = F.conv3d(_t(np.abs(x)), _t(np.abs(w)), _t(np.abs(b))).numpy()
    k = w.shape[1] * w.shape[2] * w.shape[3] * w.shape[4] + 1
    return dict(conv_fwd=ratio(np.abs(np.asarray(got) - ref), 2 * gamma(k) * ab, "conv_forward"))


def check_conv_dx(x, w, dy, got):
    ref = torch.nn.grad.conv3d_input(x.shape, _t(w), _t(dy)).numpy()
    ab = torch.nn.grad.conv3d_input(x.shape, _t(np.abs(w)), _t(np.abs(dy))).numpy()
    k = w.shape[0] * w.shape[2] * w.shape[3] * w.shape[4] + 1
    return dict(conv_dx=ratio(np.abs(np.asarray(got) - ref), 2 * gamma(k) * ab, "conv_backward dx"))


def check_conv_dw(x, w, dy, got):
    """got [Cout, Cin, kd, kh, kw]: (gamma_{ceil(R/64) + 3 + 64} + gamma_R) |x|^T |dy|."""
    ref = torch.nn.grad.conv3d_weight(_t(x), w.shape, _t(dy)).numpy()
    ab = torch.nn.grad.conv3d_weight(_t(np.abs(x)), w.shape, _t(np.abs(dy))).numpy()
    R = dy.shape[0] * dy.shape[2] * dy.shape[3] * dy.shape[4]
    g = gamma(math.ceil(R / SPLITS) + 3 + SPLITS) + gamma(R)
    return dict(conv_dw=ratio(np.abs(np.asarray(got) - ref), g * ab, "conv_backward dW"))


# ------------------------------------------------------------------------------------------------ running statistics
def running_bound(bounds, momentum, nbt0, N):
    """(mean bound, variance bound) of a running buffer after len(bounds) updates whose batch (mean, variance) carry the
    errors ``bounds`` [(bm, bv), ...], from num_batches_tracked = nbt0 with ``momentum`` (None: cumulative average)."""
    bm = bv = 0.0
    for k, (em, ev) in enumerate(bounds):
        m = momentum if momentum is not None else 1.0 / (nbt0 + k + 1)
        bm = bm + m * em
        bv = bv + m * ev * (N / max(N - 1, 1))
    return bm, bv


def check_running_update(rm0, rv0, nbt0, mean, var, N, momentum, rm, rv, nbt):
    """One running update of a BatchNorm (torch's rule, float64 batch statistics, fp32 buffers) against what an
    implementation stored: num_batches_tracked + 1; buffers within their fp32 storage (u32 |r|) plus the float64
    evaluation's gamma_4 of the terms."""
    assert int(nbt) == int(nbt0) + 1, "num_batches_tracked did not move by one"
    m = momentum if momentum is not None else 1.0 / (int(nbt0) + 1)
    rm0, rv0, mean, var = (np.asarray(a, np.float64) for a in (rm0, rv0, mean, var))
    corr = N / max(N - 1, 1)
    em = (1 - m) * rm0 + m * mean
    ev = (1 - m) * rv0 + m * var * corr
    bm = U32 * np.abs(em) + gamma(4) * (np.abs((1 - m) * rm0) + np.abs(m * mean))
    bv = U32 * np.abs(ev) + gamma(5) * (np.abs((1 - m) * rv0) + np.abs(m * var * corr))
    return dict(running_mean=ratio(np.abs(np.asarray(rm, np.float64) - em), bm, "running_mean"),
                running_var=ratio(np.abs(np.asarray(rv, np.float64) - ev), bv, "running_var"))


# ------------------------------------------------------------------------------------------------ module level
ETA = 1e-4          # the forward's fp32-grade bound (a8 / a11): relative to a channel's magnitude sqrt(E[x^2])
G_ELEM = 2e-5       # gradient error against the contraction on absolute values |dz|^T |x| (weights), sum |dz| (biases)
G_NORM = 1e-4       # gradient error per tensor, relative to the float64 gradient's norm
COST_CONVS = [0, 3, 6, 9, 12, 15, 18, 21, 24, 27]
BN_CONVS = COST_CONVS[:-1]
DESC_BN = ["Desc.pnt_layer.1"] + [f"Desc.conv_net.ops.{i}" for i in (1, 4, 7, 10, 13, 16, 19)] + ["Desc.pool_layer.1", "Desc.pool_layer.4"]
POSE_BN = [f"Pose.conv.ops.{i + 1}" for i in BN_CONVS]
POSE_POSITIONS = [18 * 3 * 18, 16 * 16, 14 * 14, 12 * 12, 10 * 10, 8 * 8, 6 * 6, 4 * 4, 2 * 2]   # output positions per BN layer


def bn_count(key, K):
    """The samples a BatchNorm averages over in one call with K matches.  CostNet: K x the layer's output positions.
    The descriptor network: both of its calls in a step describe the K matched key-points, one patch each (the source
    call the source key-points, the target call the target key-points of the same K matches), so each call averages over
    K x 140 positions (conv_net, pool_layer) or K x 420 x voxel_sample samples (pnt_layer).  K x 140 is the least of
    these, and the least N gives the largest N / (N - 1), so it bounds every descriptor layer."""
    if key.startswith("Pose"):
        return K * POSE_POSITIONS[POSE_BN.index(key)]
    return K * 140


def stat_bound(mean, var):
    """|batch mean error| and |batch variance error| allowed for a channel: the layer's values carry an error of at most
    ETA sqrt(E[x^2]), so the mean moves by at most that and the variance by at most 2 ETA E[x^2] (+ ETA^2 E[x^2])."""
    ex2 = var + mean * mean
    return ETA * torch.sqrt(ex2) + 1e-12, (2 * ETA + ETA * ETA) * ex2 + 1e-12


def check_batch_stats(got, ref, keys, what):
    """[(mean, var)] per BatchNorm call against the float64 oracle's -> [(mean bound, var bound)]."""
    assert len(got) == len(ref) == len(keys), what
    out = []
    for key, (gm, gv), (om, ov) in zip(keys, got, ref):
        bm, bv = stat_bound(om, ov)
        em, ev = (gm.cpu() - om).abs(), (gv.cpu() - ov).abs()
        assert (em <= bm).all(), f"{what} {key}: batch mean err {(em / bm).max()} x bound"
        assert (ev <= bv).all(), f"{what} {key}: batch var err {(ev / bv).max()} x bound"
        out.append((bm, bv))
    return out


def check_running_buffers(msd, ostate, key, bounds, momentum, nbt0, N):
    """The running buffers of BatchNorm ``key`` after len(bounds) updates against the oracle state: running_bound of the
    batch-statistic bounds plus the fp32 storage of the buffers (2^-22 |r|: a rounding per update, at most two here)."""
    bm, bv = running_bound(bounds, momentum, nbt0, N)
    for buf, b in (("running_mean", bm), ("running_var", bv)):
        g, o = msd[key + "." + buf].cpu().double(), ostate[key + "." + buf]
        err = (g - o).abs()
        lim = b + 2.0 ** -22 * o.abs()
        assert (err <= lim).all(), f"{key}.{buf}: err {(err / lim).max()} x bound"


def check_grads(costnet, params64, absb, what):
    """Every CostNet gradient elementwise within G_ELEM of the contraction on absolute values and within G_NORM of the
    float64 gradient's norm (the BatchNorm'd layers' biases: analytically zero, within G_ELEM of it) -> ratios."""
    bad, ratios = [], {}
    for i in COST_CONVS:
        for kind in ("weight", "bias"):
            k = f"ops.{i}.{kind}"
            p = getattr(costnet.ops[i], kind)
            assert p.grad is not None, k
            g, g64 = p.grad.detach().cpu().double(), params64[k].grad
            lim = G_ELEM * absb[k] + 1e-30
            e = float(((g - g64).abs() / lim).max())
            ratios[k] = e
            if e > 1.0:
                bad.append(f"{k}: elementwise err {e:.3g} x bound")
            if kind == "bias" and i in BN_CONVS:
                if not (g.abs() <= lim).all():
                    bad.append(f"{k}: the analytically zero gradient is {float(g.abs().max()):.3g}")
            else:
                n = float((g - g64).norm()) / float(g64.norm())
                ratios[k + "/norm"] = n / G_NORM
                if n > G_NORM:
                    bad.append(f"{k}: norm err {n:.3g}")
    print(what, "gradient error / bound:", {k: round(v, 3) for k, v in ratios.items()})
    assert not bad, f"{what}: " + "; ".join(bad)
    return ratios
