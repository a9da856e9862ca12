"""GPU: the Desc training step's kernels (bx_train_desc.cu) through their ops.py wrappers against float64 torch on the
device: the cylindrical convolution's forward, data and weight gradients on the fp64 tensor cores (all eight layer shapes),
the point layer's forward and backward on edge patches, the pool layer's backward below the normalisation's eps, EquiMatch's
backward, and the wrappers' refusals.  Bounds are gamma(k) |w|^T |x| contractions, as in oracle/train_step_cases.py."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U64 = 2.0 ** -53
# (Cin, Cout, Din) of Cylindrical_Net's eight convolutions (models/patchnet.py:68-84)
LAYERS = [(16, 64, 3), (64, 64, 1), (64, 128, 1), (128, 128, 1), (128, 64, 1), (64, 64, 1), (64, 32, 1), (32, 32, 1)]
KS = (1, 2, 3, 37, 512)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def _ops():
    from bufferx_b200 import ops
    return ops


def _blk(x):
    """[n, C, S] -> blocked [n, C/4, S, 4]"""
    n, C, S = x.shape
    return x.view(n, C // 4, 4, S).permute(0, 1, 3, 2).contiguous()


def _unblk(x):
    n, G, S, _ = x.shape
    return x.permute(0, 1, 3, 2).reshape(n, 4 * G, S)


def _pad_cyl(x):
    x = torch.cat([x[..., -1:], x, x[..., :1]], dim=-1)
    return F.pad(x, [0, 0, 1, 1])


def _wide(shape, seed, dev):
    """values over ~12 decades, both signs, some exact zeros"""
    g = torch.Generator().manual_seed(seed)
    m = torch.randn(shape, generator=g, dtype=torch.float64)
    e = torch.randint(-6, 7, shape, generator=g).double()
    v = m * 10.0 ** e
    v[torch.rand(shape, generator=g) < 0.05] = 0.0
    return v.to(dev)


def _conv_ref(x5, w, b, Din):
    """x5 [n, Cin, Din, 7, 20] -> F.conv3d on the padded input [n, Cout, 7, 20]"""
    return F.conv3d(_pad_cyl(x5), w, b).squeeze(2)


@pytest.mark.parametrize("K", KS)
@pytest.mark.parametrize("layer", range(8))
def test_cyl_conv_matches_float64(dev, layer, K):
    ops = _ops()
    Cin, Cout, Din = LAYERS[layer]
    x5 = _wide((K, Cin, Din, 7, 20), 10 * layer + K, dev)
    w = _wide((Cout, Cin, Din, 3, 3), 7 + layer, dev) * 1e-3
    b = _wide((Cout,), 3 + layer, dev)
    dy = _wide((K, Cout, 7, 20), 99 + layer + K, dev)
    xb = _blk(x5.reshape(K, Cin, Din * 140))
    Wt = w.reshape(Cout, Cin, -1).permute(2, 1, 0).contiguous()
    k = Din * 9 * Cin
    # forward
    got = _unblk(ops.cyl_forward(xb, Wt, b, Din)).view(K, Cout, 7, 20)
    ref = _conv_ref(x5, w, b, Din)
    bound = 1.01 * k * U64 / (1 - k * U64) * (_conv_ref(x5.abs(), w.abs(), b.abs(), Din)) + 1e-300
    assert ((got - ref).abs() <= bound).all(), f"forward err {float(((got - ref).abs() / bound).max())} x bound"
    # data and weight gradients
    dyb = _blk(dy.reshape(K, Cout, 140))
    dx, dW = ops.cyl_backward(xb, dyb, Wt, Din)
    xr = x5.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    _conv_ref(xr, wr, b, Din).backward(dy)
    xa = x5.abs().requires_grad_(True)
    wa = w.abs().requires_grad_(True)
    _conv_ref(xa, wa, None, Din).backward(dy.abs())
    kd = 9 * Cout
    got_dx = _unblk(dx).view(K, Cin, Din, 7, 20)
    bdx = 1.01 * kd * U64 / (1 - kd * U64) * xa.grad + 1e-300
    assert ((got_dx - xr.grad).abs() <= bdx).all(), f"dgrad err {float(((got_dx - xr.grad).abs() / bdx).max())} x bound"
    kw = K * 140
    got_dw = dW.permute(2, 1, 0).reshape(w.shape)
    bdw = 1.01 * kw * U64 / (1 - kw * U64) * wa.grad + 1e-300
    assert ((got_dw - wr.grad).abs() <= bdw).all(), f"wgrad err {float(((got_dw - wr.grad).abs() / bdw).max())} x bound"
    _, dW2 = ops.cyl_backward(xb, dyb, Wt, Din, want_dx=False)
    assert torch.equal(dW, dW2)                  # fixed split order: bit-identical


def _pnt_case(kind, dev, K=6, V=420, nv=10, seed=0):
    g = torch.Generator().manual_seed(seed)
    inv = (torch.randn((K, V, nv, 3), generator=g) * 0.3).float()
    inv[:, :, 7:] = 0.0                                           # zero slots
    W = torch.randn((16, 3), generator=g, dtype=torch.float64)
    b = torch.randn(16, generator=g, dtype=torch.float64) * 0.1
    gamma = torch.rand(16, generator=g, dtype=torch.float64) + 0.5
    beta = torch.randn(16, generator=g, dtype=torch.float64) * 0.2
    if kind == "zero_patch":
        inv[0] = 0.0                                              # every sample ties at the bias
    elif kind == "ties":
        inv[:, :, 1] = inv[:, :, 0]                               # an exact duplicate of the first sample
        beta += 1.0                                               # positive, so the tie is a maximum that passes the ReLU
    elif kind == "zero_var":
        W[3] = 0.0                                                # channel 3: y = b, zero batch variance
    return inv.to(dev), W.to(dev), b.to(dev), gamma.to(dev), beta.to(dev)


@pytest.mark.parametrize("kind", ["random", "zero_patch", "ties", "zero_var"])
def test_point_layer_matches_float64(dev, kind):
    ops = _ops()
    inv, W, b, gamma, beta = _pnt_case(kind, dev)
    K, V, nv, _ = inv.shape
    eps = 1e-5
    x = inv.double()
    y = x @ W.t() + b                                              # [K, V, nv, 16]
    mean = y.mean(dim=(0, 1, 2))
    var = y.var(dim=(0, 1, 2), unbiased=False)
    rstd = 1.0 / torch.sqrt(var + eps)
    scale = (gamma * rstd).contiguous()
    shift = (beta - mean * scale).contiguous()
    feat, arg = ops.pnt_forward(inv, W.contiguous(), b.contiguous(), scale, shift)
    r = torch.relu(y * scale + shift)
    ref, ref_arg = F.max_pool2d(r.permute(0, 3, 1, 2), kernel_size=(1, nv), return_indices=True)
    got = _unblk(feat).view(K, 16, V)
    assert (got - ref[..., 0]).abs().max() <= 1e-12 * max(1.0, float(ref.abs().max()))
    assert torch.equal(arg.long(), ref_arg[..., 0] % nv)            # the first maximal sample
    # backward against autograd through the batch statistics
    Wr, br, gr, bt = (t.clone().requires_grad_(True) for t in (W, b, gamma, beta))
    yr = x @ Wr.t() + br
    xh = F.batch_norm(yr.permute(0, 3, 1, 2), None, None, gr, bt, training=True, eps=eps)
    out = F.max_pool2d(torch.relu(xh), kernel_size=(1, nv))[..., 0]
    dfeat = torch.randn(out.shape, dtype=torch.float64, device=dev)
    out.backward(dfeat)
    o = ops.pnt_backward(inv, arg, _blk(dfeat), W.contiguous(), b.contiguous(), mean.contiguous(), rstd.contiguous(),
                         gamma.contiguous(), scale, shift, ops.moments3(inv))
    # bounds: the sums over the R samples on absolute values
    R = K * V * nv
    xa = x.abs().reshape(R, 3)
    dza = torch.zeros((K, 16, V, nv), dtype=torch.float64, device=dev)
    dza.scatter_(3, arg.long().unsqueeze(3), dfeat.abs().unsqueeze(3))
    dza = dza.permute(0, 2, 3, 1).reshape(R, 16)
    G = (gamma * rstd).abs()
    lim_w = 1e-9 * G[:, None] * (dza.t() @ xa + dza.sum(0)[:, None] * xa.mean(0)[None] * 3)
    for got_g, ref_g, lim, what in ((o[:, :3], Wr.grad, lim_w, "dW"), (o[:, 4], gr.grad, 1e-9 * (dza.sum(0) * 10 + 1e-300), "dgamma"),
                                    (o[:, 5], bt.grad, 1e-9 * (dza.sum(0) + 1e-300), "dbeta"),
                                    (o[:, 3], br.grad, 1e-9 * G * dza.sum(0) + 1e-300, "db")):
        assert ((got_g - ref_g).abs() <= lim + 1e-12 * ref_g.abs()).all(), f"{kind} {what}: {float((got_g - ref_g).abs().max())}"


def _pool_ref(x, w):
    f = (x * w[:, None]).mean(dim=2)
    return F.normalize(f, dim=1), F.normalize(x, dim=1)


@pytest.mark.parametrize("K", [1, 5, 64])
def test_pool_layer_backward_below_eps(dev, K):
    ops = _ops()
    g = torch.Generator().manual_seed(K)
    x = torch.randn((K, 32, 140), generator=g, dtype=torch.float64)
    w = torch.relu(torch.randn((K, 140), generator=g, dtype=torch.float64))
    w[0] = 0.0                                                     # all-zero attention: |desc| below eps
    x[0, :, 5] = 0.0                                               # zero-norm equi positions
    x[-1, :, 17] = 1e-14
    x, w = x.to(dev), w.to(dev)
    wb = torch.zeros((K, 1, 140, 4), dtype=torch.float64, device=dev)
    wb[:, 0, :, 0] = w
    f, desc, equi = ops.pool_forward(_blk(x), wb)
    rd, re = _pool_ref(x, w)
    assert (desc.double() - rd).abs().max() < 1e-6 and (equi.double().view(K, 32, 140) - re).abs().max() < 1e-6
    ddesc = torch.randn((K, 32), device=dev).float()
    dequi = torch.randn((K, 32, 7, 20), device=dev).float()
    dx, dw = ops.pool_backward(_blk(x), wb, f, ddesc, dequi)
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    d, e = _pool_ref(xr, wr)
    torch.autograd.backward([d, e], [ddesc.double(), dequi.double().view(K, 32, 140)])
    gx, gw = _unblk(dx), dw[:, 0, :, 0]
    assert torch.allclose(gx, xr.grad, rtol=1e-10, atol=1e-10 * float(xr.grad.abs().max())), float((gx - xr.grad).abs().max())
    assert torch.allclose(gw, wr.grad, rtol=1e-10, atol=1e-10 * float(wr.grad.abs().max()) + 1e-300)
    assert (dw[:, 0, :, 1:] == 0).all()


@pytest.mark.parametrize("B", [1, 3, 512])
def test_equi_match_backward(dev, B):
    ops = _ops()
    s = torch.randn((B, 32, 7, 20), device=dev)
    t = torch.randn((B, 32, 7, 20), device=dev)
    dcor = torch.randn((B, 20), device=dev)
    gs, gt = ops.equi_match_backward(s, t, dcor)
    sr, tr = s.double().requires_grad_(True), t.double().requires_grad_(True)
    L = 20
    idx = (torch.arange(L)[None, :] - torch.arange(L)[:, None]) % L
    cor = torch.einsum("kceal,kcel->ka", sr[..., idx.to(dev)], tr)
    cor.backward(dcor.double())
    assert torch.allclose(cor.float(), ops.equi_match(s, t), rtol=1e-4, atol=1e-3)
    assert (gs.double() - sr.grad).abs().max() <= 1e-6 * float(sr.grad.abs().max())
    assert (gt.double() - tr.grad).abs().max() <= 1e-6 * float(tr.grad.abs().max())


def test_desc_wrappers_refuse_misshaped_inputs(dev):
    ops = _ops()
    x = torch.zeros((2, 4, 420, 4), dtype=torch.float64, device=dev)
    Wt = torch.zeros((27, 16, 64), dtype=torch.float64, device=dev)
    b = torch.zeros(64, dtype=torch.float64, device=dev)
    with pytest.raises(ops.BufferXError):
        ops.cyl_forward(x, Wt, b, 1)                               # 420 positions, not one slice
    with pytest.raises(ops.BufferXError):
        ops.cyl_forward(x.float(), Wt, b, 3)
    with pytest.raises(ops.BufferXError):
        ops.cyl_forward(x, Wt[:, :, :60], b, 3)
    with pytest.raises(ops.BufferXError):
        ops.cyl_backward(x, torch.zeros((2, 16, 140, 4), dtype=torch.float64, device=dev)[:, :8], Wt, 3)
    inv = torch.zeros((2, 420, 10, 3), device=dev)
    v16 = torch.zeros(16, dtype=torch.float64, device=dev)
    with pytest.raises(ops.BufferXError):
        ops.pnt_forward(inv[..., :2], torch.zeros((16, 3), dtype=torch.float64, device=dev), v16, v16, v16)
    with pytest.raises(ops.BufferXError):
        ops.pnt_forward(inv, torch.zeros((16, 4), dtype=torch.float64, device=dev), v16, v16, v16)
    with pytest.raises(ops.BufferXError):
        ops.pool_forward(torch.zeros((2, 8, 139, 4), dtype=torch.float64, device=dev), torch.zeros((2, 1, 139, 4), dtype=torch.float64, device=dev))
    with pytest.raises(ops.BufferXError):
        ops.equi_match_backward(torch.zeros((2, 32, 7, 20), device=dev), torch.zeros((2, 32, 7, 20), device=dev), torch.zeros((2, 19), device=dev))
    with pytest.raises(ops.BufferXError):
        ops.conv1x1(torch.zeros((2, 8, 140, 4), dtype=torch.float64, device=dev), torch.zeros((32, 36), dtype=torch.float64, device=dev))
