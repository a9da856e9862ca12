"""GPU: every kernel of the Pose training step (csrc/bx_train_step.cu), called through its ops.py wrapper, against the
float64 checks of oracle/train_step_cases.py (the bounds are derived there) on edge shapes and inputs; the wrappers'
refusals; the point layer's moment-derived batch statistics; CostNet's training forward + backward at M in {1, 2, 3, 65}, with momentum None and eps 1e-3 over two steps,
and with a non-finite map.  The worst ratio of every check is printed with -s and recorded in DESIGN.md section 7."""

import numpy as np
import pytest
import torch

from oracle import train_desc_cases as D
from oracle import train_step_cases as C

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bx():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return bx


def _cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(t):
    torch.cuda.synchronize()
    return t.detach().cpu().numpy()


# ------------------------------------------------------------------------------------------------ channel sums
def _sum_shapes():
    out = [(n, S, 4) for n in C.SUM_N for S in C.SUM_S]
    return out + [(n, S, Cc) for Cc in (20, 128) for n in (1, 65) for S in (257, 972)]


def test_channel_sums(bx):
    acc = {}
    for i, (n, S, Cc) in enumerate(_sum_shapes()):
        for kind, dt in ((k, d) for k in ("const", "positive", "offset") for d in (np.float32, np.float64)):
            x = C.sums_input(n, Cc, S, kind, seed=i, dtype=dt)
            xb = _cu(C.to_blocked(x))
            got = bx.ops.channel_sums(xb)
            C.merge(acc, C.check_channel_sums(x, _np(got)))
            assert torch.equal(got, bx.ops.channel_sums(xb)), "two calls differ"
    C.report("channel_sums (fp32 + f64)", acc)


def test_bn_backward_at_gamma_1_on_mask_edges(bx):
    """The BatchNorm + ReLU backward with gamma = 1 (the affine = False layers of CostNet and Cylindrical_Net: rstd = scale)
    held to check_bn_affine_backward on mask_case's edge inputs; the forward is bn_apply_f64 with ReLU, and the backward
    takes its output y as the mask."""
    acc = {}
    for n, S, Cc in _sum_shapes():
        dy, z, sc, sh, mean = C.mask_case(n, Cc, S, seed=n + S)
        xh = C.xhat(z, sc, sh)
        dyb, zb = _cu(C.to_blocked(dy)), _cu(C.to_blocked(z))
        scb, meanb, gam = _cu(sc), _cu(mean), torch.ones(Cc, dtype=torch.float64, device="cuda")
        yb = bx.ops.bn_apply(zb, scb, _cu(sh), True)
        y = C.from_blocked(_np(yb))
        C.check_mask(z, sc, sh, y > 0, xh)
        _, cnt = bx.ops.bn_backward(torch.ones_like(zb), zb, yb, meanb, scb, gam)
        assert np.array_equal(_np(cnt)[0], (y > 0).sum(axis=(0, 2)).astype(np.float64)), "bn_backward's sums count another mask"
        dx, s = bx.ops.bn_backward(dyb, zb, yb, meanb, scb, gam)
        C.merge(acc, D.check_bn_affine_backward(dy, z, y, mean, sc, np.ones(Cc), C.from_blocked(_np(dx)), _np(s)))
        dx2, s2 = bx.ops.bn_backward(dyb, zb, yb, meanb, scb, gam)
        assert torch.equal(s, s2) and torch.equal(dx, dx2), "two calls differ"
    C.report("bn mask / bn_backward at gamma = 1", acc)


def test_bn_apply(bx):
    acc = {}
    for n, S, Cc in ((1, 1, 4), (2, 7, 12), (65, 257, 20), (3, 2001, 128)):
        for dt in (np.float32, np.float64):
            z, sc, sh = C.apply_case(n, Cc, S, seed=S, dtype=dt)
            for relu in (False, True):
                y = bx.ops.bn_apply(_cu(C.to_blocked(z)), _cu(sc), _cu(sh), relu)
                C.merge(acc, C.check_bn_apply(z, sc, sh, relu, C.from_blocked(_np(y))))
    C.report("bn_apply", acc)


def test_moments3(bx):
    acc = {}
    for R in C.MOM_R:
        for off in (0.0, 1e3):
            v = C.moments_input(R, off, seed=R)
            C.merge(acc, C.check_moments3(v, _np(bx.ops.moments3(_cu(v)))))
    C.report("moments3", acc)


def test_point_layer_stats_from_moments(bx):
    """moments3 + pnt_stats_from_moments (the point layer's batch statistics) against a float64 BatchNorm over the explicit
    point-layer outputs; coordinates offset by 1e3 make E[x x^T] ~ 1e6 cancel to a covariance of ~0.1."""
    from bufferx_b200.models.patch_embedder import pnt_stats_from_moments
    acc = {}
    rng = np.random.default_rng(6)
    W, b = rng.normal(size=(16, 3)) * 0.7, rng.normal(size=16) * 0.1
    for K, off in ((1, 0.0), (64, 0.0), (3, 1e3), (65, 1e3), (7, 10.0)):
        inv = C.pnt_inv_case(K, off, seed=K)
        mo = bx.ops.moments3(_cu(inv)) / (inv.size // 3)
        mean, var = pnt_stats_from_moments(mo, _cu(W), _cu(b))
        C.merge(acc, C.check_pnt_stats(inv, W, b, _np(mean), _np(var)))
    C.report("point layer stats from moments", acc)


def test_point_layer_stats_in_the_training_step(bx, monkeypatch):
    """MiniSpinNet.forward_train inside a Pose step (source and target calls): the point layer's batch statistics it
    records against a float64 BatchNorm over the point-layer outputs of the very samples it took the moments of."""
    from bufferx_b200.synth import add_training_clouds, init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C1")
    cfg.stage = "Pose"
    cfg.train.pos_num = 64
    data = add_training_clouds(make_pair("C1", 0), cfg)
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True).cuda()
    for p in model.Desc.parameters():
        p.requires_grad = False
    seen = []
    orig = bx.ops.moments3

    def spy(v):
        seen.append(v.detach().cpu().numpy().copy())
        return orig(v)
    monkeypatch.setattr(bx.ops, "moments3", spy)
    model.train()
    np.random.seed(4)
    model(data)
    assert len(seen) == 2
    W = model.Desc.pnt_layer[0].weight.detach().double().view(16, 3).cpu().numpy()
    b = model.Desc.pnt_layer[0].bias.detach().double().cpu().numpy()
    acc = {}
    for side, inv in zip(("src", "tgt"), seen):
        mean, var = model.last_train_stats[side][0]
        C.merge(acc, C.check_pnt_stats(inv, W, b, _np(mean), _np(var)))
    C.report("point layer stats in the step", acc)


def test_conv1x1(bx):
    acc = {}
    rng = np.random.default_rng(5)
    for Cin in (4, 16, 32):
        for Cout4 in (4, 8, 12, 16):
            for n, S in ((1, 7), (65, 141)):
                x = rng.normal(size=(n, Cin, S)).astype(np.float32)
                w = rng.normal(size=(Cin, Cout4)).astype(np.float32)
                b = rng.normal(size=Cout4).astype(np.float32)
                w[:, -1], b[-1] = 0, 0                      # a zero-padded output channel
                y = bx.ops.conv1x1(_cu(C.to_blocked(x)), _cu(w), _cu(b))
                C.merge(acc, C.check_conv1x1(x, w, b, C.from_blocked(_np(y))))
    C.report("conv1x1", acc)


def test_costvol(bx):
    acc = {}
    for M in C.COSTVOL_M:
        for wide in (False, True):
            s, t = C.costvol_maps(M, seed=M, wide=wide)
            C.merge(acc, C.check_costvol(s, t, _np(bx.ops.costvol(_cu(s), _cu(t)))))
    C.report("costvol", acc)


def test_softargmax(bx):
    acc = {}
    for L in C.SAM_L:
        for M in C.SAM_M:
            for kind in ("flat", "spread", "tied", "huge", "offset", "normal"):
                lg = C.sam_logits(M, L, kind, seed=M + L)
                g = np.random.default_rng(M).normal(size=M)
                g[::5] = 0.0
                C.merge(acc, C.check_softargmax(lg, _np(bx.ops.softargmax(_cu(lg)))))
                C.merge(acc, C.check_softargmax_backward(lg, g, _np(bx.ops.softargmax(_cu(lg), _cu(g)))))
    C.report("softargmax", acc)


def test_softargmax_nonfinite_row(bx):
    lg = C.sam_logits(129, 20, "normal", seed=3)
    g = np.random.default_rng(3).normal(size=129)
    ref_i, ref_d = _np(bx.ops.softargmax(_cu(lg))), _np(bx.ops.softargmax(_cu(lg), _cu(g)))
    for bad in (np.inf, np.nan):
        lb = lg.copy()
        lb[64, 7] = bad
        i, d = _np(bx.ops.softargmax(_cu(lb))), _np(bx.ops.softargmax(_cu(lb), _cu(g)))
        assert not np.isfinite(i[64]) and not np.isfinite(d[64]).all()
        keep = np.arange(129) != 64
        assert np.array_equal(i[keep], ref_i[keep]) and np.array_equal(d[keep], ref_d[keep])


# ------------------------------------------------------------------------------------------------ convolutions
def _conv_cases():
    out = []
    for li, (Cin, Cout, DHW, k) in enumerate(C.COSTNET_GEOMS):
        for M in (1, 2, 3, 63, 64, 65):
            out.append((f"L{li}_M{M}", M, Cin, Cout, DHW, k))
    for j, (n, Cin, Cout, DHW, k) in enumerate(C.SYNTH_GEOMS):
        out.append((f"synth{j}", n, Cin, Cout, DHW, k))
    return out


def _blk(a):
    """[n, C, D, H, W] -> blocked [n, C/4, D*H*W, 4] on the GPU."""
    return _cu(C.to_blocked(a.reshape(a.shape[0], a.shape[1], -1)))


def _unblk(t, shape):
    return C.from_blocked(_np(t)).reshape(shape)


def test_conv_forward_and_backward(bx):
    acc = {}
    for j, (name, n, Cin, Cout, (D, H, W), (kd, kh, kw)) in enumerate(_conv_cases()):
        x, w, b, dy = C.conv_case(n, Cin, Cout, (D, H, W), (kd, kh, kw), seed=j)
        xb, dyb, Wt = _blk(x), _blk(dy), _cu(C.wt_of(w))
        y = bx.ops.conv_forward(xb, Wt, _cu(b), D, H, W, kd, kh, kw)
        C.merge(acc, C.check_conv_forward(x, w, b, _unblk(y, dy.shape)))
        dx, dW = bx.ops.conv_backward(xb, dyb, Wt, D, H, W, kd, kh, kw)
        C.merge(acc, C.check_conv_dx(x, w, dy, _unblk(dx, x.shape)))
        dWn = _np(dW).transpose(2, 1, 0).reshape(w.shape)
        C.merge(acc, C.check_conv_dw(x, w, dy, dWn))
        dx2, dW2 = bx.ops.conv_backward(xb, dyb, Wt, D, H, W, kd, kh, kw, want_dx=False)
        assert dx2 is None and torch.equal(dW2, dW), f"{name}: want_dx=False changed dW"
    C.report("conv_forward / conv_backward", acc)


# ------------------------------------------------------------------------------------------------ refusals
def test_wrapper_refusals(bx):
    ops, E = bx.ops, bx.ops.BufferXError
    f64 = dict(dtype=torch.float64, device="cuda")
    x = torch.zeros((1, 8, 4 * 1 * 4, 4), **f64)
    with pytest.raises(E):                                 # Cin % 32
        ops.conv_forward(torch.zeros((1, 4, 16, 4), **f64), torch.zeros((9, 16, 4), **f64), torch.zeros(4, **f64), 4, 1, 4, 3, 1, 3)
    with pytest.raises(E):                                 # Cout % 4
        ops.conv_forward(x, torch.zeros((9, 32, 6), **f64), torch.zeros(6, **f64), 4, 1, 4, 3, 1, 3)
    with pytest.raises(E):                                 # kernel larger than the extent
        ops.conv_forward(x, torch.zeros((5, 32, 4), **f64), torch.zeros(4, **f64), 4, 1, 4, 5, 1, 1)
    with pytest.raises(E):                                 # M = 0
        ops.conv_forward(torch.zeros((0, 8, 16, 4), **f64), torch.zeros((9, 32, 4), **f64), torch.zeros(4, **f64), 4, 1, 4, 3, 1, 3)
    with pytest.raises(E):                                 # x holds another geometry
        ops.conv_forward(x, torch.zeros((9, 32, 4), **f64), torch.zeros(4, **f64), 4, 1, 5, 3, 1, 3)
    with pytest.raises(E):                                 # Wt of another Cin
        ops.conv_forward(x, torch.zeros((9, 64, 4), **f64), torch.zeros(4, **f64), 4, 1, 4, 3, 1, 3)
    with pytest.raises(E):                                 # dy of another output
        ops.conv_backward(x, torch.zeros((1, 1, 3, 4), **f64), torch.zeros((9, 32, 4), **f64), 4, 1, 4, 3, 1, 3)
    with pytest.raises(E):
        ops.conv_backward(x, torch.zeros((1, 1, 4, 4), **f64), torch.zeros((9, 32, 4), **f64), 4, 1, 4, 3, 1, 2)
    f32 = dict(dtype=torch.float32, device="cuda")
    for s, t in (((2, 32, 5, 20), (2, 32, 5, 20)), ((2, 32, 7, 20), (1, 32, 7, 20)), ((2, 16, 7, 20), (2, 16, 7, 20)),
                 ((0, 32, 7, 20), (0, 32, 7, 20))):
        with pytest.raises(E):
            ops.costvol(torch.zeros(s, **f32), torch.zeros(t, **f32))
    z = torch.zeros((2, 3, 5, 4), **f64)
    c12, c8 = torch.zeros(12, **f64), torch.zeros(8, **f64)
    z4 = torch.zeros((2, 3, 4, 4), **f64)
    with pytest.raises(E):
        ops.channel_sums(torch.zeros((2, 3, 5), **f64))
    for args in ((z, z, z4, c12, c12, c12), (z, z, z, c8, c12, c12), (z, z, z, c12, c8, c12), (z, z, z, c12, c12, c8),
                 (z4, z, z, c12, c12, c12)):              # y, mean, rstd, gamma, dy of another shape
        with pytest.raises(E):
            ops.bn_backward(*args)
    with pytest.raises(E):                                 # the backward takes float64 only
        ops.bn_backward(z.float(), z.float(), z.float(), c12.float(), c12.float(), c12.float())
    with pytest.raises(E):                                 # z of another dtype than dy
        ops.bn_backward(z, z.float(), z, c12, c12, c12)
    with pytest.raises(E):
        ops.bn_apply(z, c8, c12, True)
    with pytest.raises(E):
        ops.softargmax(torch.zeros((5, 20), **f64), torch.zeros(4, **f64))
    with pytest.raises(E):
        ops.moments3(torch.zeros((5, 2), **f32))
    with pytest.raises(E):
        ops.conv1x1(torch.zeros((1, 2, 3, 4), **f32), torch.zeros((4, 4), **f32), torch.zeros(4, **f32))
    with pytest.raises(E):                                 # Cout above 32
        ops.conv1x1(torch.zeros((1, 2, 3, 4), **f32), torch.zeros((8, 36), **f32), torch.zeros(36, **f32))
    with pytest.raises(E):                                 # w of another dtype than x
        ops.conv1x1(torch.zeros((1, 2, 3, 4), **f32), torch.zeros((8, 4), **f64))


# ------------------------------------------------------------------------------------------------ CostNet, module level
@pytest.fixture(scope="module")
def costnet(bx):
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    model = init_synthetic_weights(bx.BufferX(workload_cfg("C1")), trained_pose=True)
    return model


def _maps(M, seed):
    rng = np.random.default_rng(seed)
    return [torch.from_numpy((rng.normal(size=(M, 32, 7, 20)) * 0.3).astype(np.float32)) for _ in range(2)]


def _gt(M, seed):
    return torch.from_numpy(np.random.default_rng(seed + 7).uniform(0, 20, M).astype(np.float32))


def _gpu_step(conv, es, et, gt):
    stats = []
    conv.zero_grad(set_to_none=True)
    pred = conv.forward_train(es.cuda(), et.cuda(), stats)
    torch.nn.HuberLoss()(pred, gt.cuda()).backward()
    return pred, stats


def _oracle_step(TP, params, st, hp, es, et, gt):
    stats, keep = [], {}
    pred = TP.costnet_train(es[:, :, 1:6], et[:, :, 1:6], params, st, stats, hp, keep)
    torch.nn.functional.huber_loss(pred, gt.double()).backward()
    return pred, stats, keep


def _run_costnet(bx, oracle, model, M, steps, momentum="keep", eps=None, seed=0):
    import copy
    from oracle import train_step as TP
    m = copy.deepcopy(model)
    for i in C.BN_CONVS:
        bn = m.Pose.conv.ops[i + 1]
        if momentum != "keep":
            bn.momentum = momentum
        if eps is not None:
            bn.eps = eps
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    hp = TP.bn_hparams(m)
    m = m.cuda().train()
    conv = m.Pose.conv
    st = TP.state64(sd0)
    bounds = {k: [] for k in C.POSE_BN}
    acc = {}
    for step in range(steps):
        es, et = _maps(M, seed + step)
        gt = _gt(M, seed + step)
        params = TP.pose_params({"Pose.conv." + k: v.cpu() for k, v in conv.state_dict().items()})
        pred, stats = _gpu_step(conv, es, et, gt)
        p64, s64, keep = _oracle_step(TP, params, st, hp, es, et, gt)
        ind64, bound, _, _ = oracle.soft_argmax_bound(keep["logits"], keep["logits"].float())
        err = (pred.detach().cpu().double() - ind64).abs()
        assert (err <= torch.clamp(bound, min=1e-4)).all(), f"M={M} step {step}: pred_ind err {err.max()}"
        for key, b in zip(C.POSE_BN, C.check_batch_stats(stats, s64, C.POSE_BN, f"M={M} step {step}")):
            bounds[key].append(b)
        msd = m.state_dict()
        for key in C.POSE_BN:
            mom, _ = hp[key]
            C.check_running_buffers(msd, st, key, bounds[key], mom, int(sd0[key + ".num_batches_tracked"]), C.bn_count(key, M))
            assert int(msd[key + ".num_batches_tracked"]) == int(sd0[key + ".num_batches_tracked"]) + step + 1
        acc = C.merge(acc, C.check_grads(conv, params, TP.grad_abs_bounds(keep, params), f"M={M} step {step}"))
        with torch.no_grad():                      # the next step starts from the oracle's weights: the same for both
            for i in C.COST_CONVS:
                conv.ops[i].weight.copy_(params[f"ops.{i}.weight"].detach().float() - 1e-3 * params[f"ops.{i}.weight"].grad.float())
                conv.ops[i].bias.copy_(params[f"ops.{i}.bias"].detach().float() - 1e-3 * params[f"ops.{i}.bias"].grad.float())
    return acc


@pytest.mark.parametrize("M", [1, 2, 3, 65])
def test_costnet_train_small_batches(bx, oracle, costnet, M):
    """At M = 1 the last BatchNorm averages over N = 4 positions, so its running variance carries N / (N - 1) = 4/3."""
    acc = _run_costnet(bx, oracle, costnet, M, steps=1, seed=M)
    C.report(f"CostNet step M={M} (gradient err / bound)", {k: v for k, v in acc.items() if "norm" not in k and v == max(acc.values())})


def test_costnet_train_cumulative_average(bx, oracle, costnet):
    """momentum=None (the cumulative average, 1 / num_batches_tracked) and eps=1e-3 on every CostNet BatchNorm, two steps."""
    _run_costnet(bx, oracle, costnet, 3, steps=2, momentum=None, eps=1e-3, seed=11)


def test_costnet_nonfinite_map_gives_nonfinite_gradient(bx, costnet):
    """An inf in a map reaches the gradient of Pose.conv as a non-finite value (as in the reference), so the Trainer's
    finite check skips the step."""
    import copy
    m = copy.deepcopy(costnet).cuda().train()
    es, et = _maps(5, 3)
    es[2, 4, 3, 7] = float("inf")
    _gpu_step(m.Pose.conv, es, et, _gt(5, 3))
    assert any((~torch.isfinite(p.grad)).any() for p in m.Pose.conv.parameters())
