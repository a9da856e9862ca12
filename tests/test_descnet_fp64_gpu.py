"""The descriptor network (a6-a9) on the GPU against float64, kernel by kernel, on the route production runs.

Production (BufferX without early exit or debug) describes all jobs of a pair with MiniSpinNet.forward_multi: SPT + point
layer write the presplit fp16 image (bx_spt_pnt_sd), the first Cylindrical_Net layer reads it as a 3-chunk CYL3D input,
layers 1-6 hand presplit images on, the last writes fp32, then bx_pool_desc.  The debug route (MiniSpinNet.forward) feeds
fp32 features to the first layer instead, and the TF32 kernels take over when an activation leaves fp16 range.

Floating-point results are compared elementwise with the same operation evaluated in float64 on the same inputs:
|got - ref| <= KAPPA * absref, where absref is that operation in float64 with |x|, |W| and |b|, so that a small output (an
edge position, a weak channel, a near-zero pre-ReLU sum) cannot hide behind a max-normalised error.  KAPPA = 2e-5, as for
CostNet (tests/test_costnet_fp64_gpu.py).  The voxel selection is integer and is held bit for bit to oracle.spt.  The
float64 references run through torch's own float64 kernels on the GPU.  The largest ratio of each test is printed (run with
-s) and recorded in DESIGN.md section 7."""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import spt_cases

pytestmark = pytest.mark.gpu

KAPPA = 2e-5


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def report(name, value):
    print(f"\n[descnet-fp64] {name}: {value:.3g}")


def check(name, got, ref, absref, kappa=KAPPA):
    """Elementwise |got - ref| <= kappa * absref (same shape); returns the largest ratio."""
    got = got.to(ref.device)
    err = (got.double() - ref).abs()
    ratio = float((err / absref.clamp(min=1e-30)).max())
    bad = err > kappa * absref
    assert torch.isfinite(got).all(), f"{name}: non-finite output"
    assert not bad.any(), f"{name}: {int(bad.sum())} elements beyond {kappa} * absref, worst ratio {ratio:.3g}"
    return ratio


def nan_fp16(shape, dev):
    return torch.full(shape, float("nan"), dtype=torch.float16, device=dev)


def spt_sd_into(delta, prep, img, flag=None, w=None, b=None, nv=10, rho=0.8 / 3):
    """bx_spt_pnt_sd into a caller-owned image (so that what it leaves alone can be checked)."""
    from bufferx_b200 import ops
    K, P, _ = delta.shape
    w = prep["w_pnt"] if w is None else w
    b = prep["b_pnt"] if b is None else b
    ops._check(ops.load_library().bx_spt_pnt_sd(ops._dp(delta, torch.float32), K, P, ops._dp(prep["voxels"]), 420, 20,
                                                ops._dp(prep["rot"]), float(rho), nv, ops._dp(w), ops._dp(b), ops._dp(img),
                                                img.shape[2], ops._dp(flag), None), "bx_spt_pnt_sd")
    return img


def x48(feat):
    """[K,16,420] point-layer features -> [K,48,7,20]: 16-channel chunk r = radial slice r (the CYL3D presplit input)."""
    K = feat.shape[0]
    return feat.reshape(K, 16, 3, 140).permute(0, 2, 1, 3).reshape(K, 48, 7, 20)


# ------------------------------------------------------------------------------------------------ the C2 pair, seed 0
@pytest.fixture(scope="module")
def c2(dev, oracle):
    """A C2 pair described on the production route: the six (cloud, scale) jobs through forward_multi (9000 patches), the
    patches, oracle.spt's selection and the float64 point-layer features; the model's own batched pass gives the same bits."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, make_pair, workload_cfg
    cfg = workload_cfg("C2")
    assert cfg.match.get("enable_early_exit", True) is False
    model = init_synthetic_weights(bx.BufferX(cfg), trained_pose=True)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model = model.to(dev).eval()
    data = make_pair("C2", 0)
    perms = oracle.draw_perms(cfg, data["src_fds_pcd"].shape[0], data["tgt_fds_pcd"].shape[0], 0)
    K, S = cfg.patch.num_fps, cfg.patch.num_scales
    with torch.no_grad():
        model(data, perms=perms, ransac_seed=0)                         # production: batched forward_multi
        prod_desc = model.Desc.last_multi["desc"].clone()
        model(data, perms=perms, ransac_seed=0, debug=True)
        dbg = model.last_debug
        jobs = []
        for i in range(S):
            for j, key in ((0, "src_fds_pcd"), (1, "tgt_fds_pcd")):
                jobs.append((torch.from_numpy(np.ascontiguousarray(data[key])).to(dev), dbg["kpts"][j, :K].contiguous(),
                             dbg["des_r"][i:i + 1], torch.from_numpy(np.ascontiguousarray(perms[i][j], dtype=np.int32)).to(dev)))
        aligned = bool(data["is_aligned_to_global_z"])
        outs = model.Desc.forward_multi(jobs, aligned, radii=dbg["des_r"])
    desc = model.Desc.last_multi["desc"].clone()
    assert torch.equal(desc, prod_desc), "forward_multi on the pair's jobs differs from the model's own batched pass"
    delta = torch.cat([o["patches"] for o in outs]).contiguous()
    assert delta.shape == (2 * S * K, cfg.patch.num_points_per_patch, 3)
    t0 = time.perf_counter()
    einv, evidx = oracle.spt(delta.cpu().numpy())
    t_spt = time.perf_counter() - t0
    feat64, pabs = oracle.pnt_fp64(delta, evidx, sd, absref=True)
    return dict(cfg=cfg, model=model, sd=sd, data=data, perms=perms, jobs=jobs, aligned=aligned, delta=delta, desc=desc,
                einv=einv, evidx=evidx, feat64=feat64, pabs=pabs, prep=model.Desc.prepared(dev), t_spt=t_spt)


# ------------------------------------------------------------------------------------------------ 1+2. SPT and the point layer
SPT_CASES = [(1, 10, 0.8 / 3, (3, 7, 20)), (31, 10, 0.8 / 3, (3, 7, 20)), (33, 1, 0.8 / 3, (3, 7, 20)),
             (100, 16, 0.8 / 3, (3, 7, 20)), (512, 10, 0.8 / 3, (3, 7, 20)), (1000, 10, 0.8 / 3, (3, 7, 20)),
             (512, 10, 0.1, (3, 7, 20)), (512, 16, 0.5, (3, 7, 20)), (100, 1, 0.5, (3, 7, 20)), (33, 16, 0.1, (3, 7, 20)),
             (31, 10, 0.8 / 3, (2, 5, 12)), (512, 1, 0.5, (2, 5, 12)), (100, 16, 0.1, (4, 9, 24)),
             (1000, 10, 0.8 / 3, (4, 9, 24))]


@pytest.mark.parametrize("P,nv,rho,table", SPT_CASES,
                         ids=[f"P{p}-nv{n}-rho{r:.3g}-{t[0]}x{t[1]}x{t[2]}" for p, n, r, t in SPT_CASES])
def test_spt_selection_and_point_layer_on_edge_patches(dev, oracle, c2, P, nv, rho, table):
    """bx_spt_pnt (debug outputs) on the hand-built edge patches: the selection (vidx) and the de-rotated samples (inv) bit for
    bit against oracle.spt, for P not a multiple of 32, P < 32, nv != 10, the all-bins branch of rho = 0.5 and tables other
    than 3 x 7 x 20; the fp32 features elementwise against oracle.pnt_fp64."""
    from bufferx_b200 import ops
    rad_n, ele_n, azi_n = table
    delta = spt_cases.spt_patches(P, rad_n, azi_n, ele_n, rho, seed=P + 7 * nv)
    vox = torch.from_numpy(oracle.voxel_table(rad_n, azi_n, ele_n)).to(dev)
    rot = torch.from_numpy(oracle.derot_table(azi_n)).to(dev)
    prep = c2["prep"]
    feat, vidx, inv = ops.spt_pnt(torch.from_numpy(delta).to(dev), vox, rot, rho, nv, prep["w_pnt"], prep["b_pnt"], azi_n, debug=True)
    einv, evidx = oracle.spt(delta, rad_n, azi_n, ele_n, rho, nv)
    bad = (vidx.cpu().numpy() != evidx).any(axis=2)
    assert not bad.any(), f"selection differs in {int(bad.sum())} voxels, first (patch, voxel) {np.argwhere(bad)[:4].tolist()}"
    assert (inv.cpu().numpy().view(np.int32) == einv.view(np.int32)).all(), "de-rotated samples differ"
    f64, absref = oracle.pnt_fp64(delta, evidx, c2["sd"], absref=True, azi_n=azi_n)
    r = check("point layer", ops.from_blocked(feat), f64.to(dev), absref.to(dev))
    report(f"spt P={P} nv={nv} rho={rho:.3g} table={table}: selection bit-exact, point layer", r)


def test_spt_selection_and_point_layer_on_c2_patches(dev, oracle, c2):
    """The real C2 patches (6 x 1500): selection and samples bit for bit, features elementwise."""
    from bufferx_b200 import ops
    prep = c2["prep"]
    feat, vidx, inv = ops.spt_pnt(c2["delta"], prep["voxels"], prep["rot"], 0.8 / 3, 10, prep["w_pnt"], prep["b_pnt"], 20, debug=True)
    assert (vidx.cpu().numpy() == c2["evidx"]).all()
    assert (inv.cpu().numpy().view(np.int32) == c2["einv"].view(np.int32)).all()
    r = check("point layer C2", ops.from_blocked(feat), c2["feat64"], c2["pabs"])
    report(f"spt C2 9000 patches (oracle.spt {c2['t_spt']:.2f} s on the CPU): point layer", r)


@pytest.mark.parametrize("K", [1, 2, 3, 1500])
def test_spt_presplit_image(dev, c2, K):
    """bx_spt_pnt_sd into a NaN-filled image: features within the bound after decoding, the zero row above every sample,
    the wrap columns, the zero row after the last sample; nothing past it is written; bit-identical to sd_pack of
    bx_spt_pnt's fp32 features."""
    from bufferx_b200 import ops
    prep = c2["prep"]
    delta = c2["delta"][:K].contiguous()
    rows = ops.conv_sd_rows(K)
    img = spt_sd_into(delta, prep, nan_fp16((3, 4, rows, 8), dev))
    val, xp = ops.sd_unpack(img, K)
    r = check(f"presplit K={K}", val, x48(c2["feat64"][:K]), x48(c2["pabs"][:K]))
    assert (xp[:, :, 0] == 0).all(), "zero row above the first elevation"
    assert torch.equal(xp[:, :, 1:, 0], xp[:, :, 1:, 20]) and torch.equal(xp[:, :, 1:, 21], xp[:, :, 1:, 1]), "wrap columns"
    assert (img[:, :, K * 176:K * 176 + 22] == 0).all(), "the zero row after the last sample"
    assert torch.isnan(img[:, :, K * 176 + 22:]).all(), "rows past the last sample's zero row were written"
    feat = ops.spt_pnt(delta, prep["voxels"], prep["rot"], 0.8 / 3, 10, prep["w_pnt"], prep["b_pnt"], 20)
    want = ops.sd_pack(x48(ops.from_blocked(feat)))
    n = K * 176 + 22
    assert torch.equal(img[:, :, :n].view(torch.int16), want[:, :, :n].view(torch.int16))
    report(f"spt presplit K={K}", r)


@pytest.mark.parametrize("target,flagged", [(64000.0, 0), (66000.0, 1)])
def test_spt_presplit_fp16_range_flag(dev, c2, target, flagged):
    """Point-layer weights scaled so that the largest feature of 1500 real patches is `target`: >= 65000 raises the
    fp16-range flag, 64000 does not and those values stay within the bound."""
    from bufferx_b200 import ops
    prep = c2["prep"]
    K = 1500
    delta = c2["delta"][:K].contiguous()
    s = target / float(c2["feat64"][:K].max())
    w, b = (prep["w_pnt"].double() * s).float(), (prep["b_pnt"].double() * s).float()
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    img = spt_sd_into(delta, prep, nan_fp16((3, 4, ops.conv_sd_rows(K), 8), dev), flag, w, b)
    assert int(flag.item()) == flagged
    val, _ = ops.sd_unpack(img, K)
    if flagged:                       # fp16 hi saturates to inf: the image is unusable, which is what the flag reports
        assert not torch.isfinite(val).all()
    else:
        assert abs(float(val.max()) - target) <= 1e-3 * target
        r = check("presplit at 64000", val, x48(c2["feat64"][:K]) * s, x48(c2["pabs"][:K]) * s)
        report("spt presplit, largest feature 64000 (no flag)", r)


# ------------------------------------------------------------------------------------------------ 3. the eight layers
def w5(Wt, k):
    """Folded [T, Cin, Cout] -> float64 conv weight [Cout, Cin, *k]."""
    return Wt.detach().double().permute(2, 1, 0).reshape(Wt.shape[2], Wt.shape[1], *k)


def layer64(x, l, first):
    """(out, absref) of one folded Cylindrical_Net layer in float64: x [K,16,3,7,20] (first) or [K,Cin,7,20]."""
    from oracle.oracle import _pad_cyl
    W, b = w5(l["w"], l["k"]).to(x.device), l["b"].double().to(x.device)
    if not first:
        W = W[:, :, 0]
    conv = F.conv3d if first else F.conv2d
    xp = _pad_cyl(x)
    out, absref = conv(xp, W, b), conv(xp.abs(), W.abs(), b.abs())
    if first:
        out, absref = out.squeeze(2), absref.squeeze(2)
    return (torch.relu(out) if l["relu"] else out), absref


def random_layers(L, dev):
    """The eight layer shapes with seeded random weights (std 1 / sqrt(fan-in)) and biases."""
    g = torch.Generator().manual_seed(8)
    from bufferx_b200 import ops
    out = []
    for l in L:
        T, Cin, Cout = l["w"].shape
        W = (torch.randn(T, Cin, Cout, generator=g) / (T * Cin) ** 0.5).to(dev)
        out.append(dict(l, w=W, b=(0.1 * torch.randn(Cout, generator=g)).to(dev), w_sd=ops.conv_sd_weights(W),
                        w_tc=ops.conv_tc_weights(W)))
    return out


@pytest.fixture(scope="module")
def chain(dev, oracle, c2):
    """Per variant: the folded layers and the input of every layer (fp32) with its float64 output and absref, 9000 patches.
    Layer 0's input is the GPU point-layer features (what both routes feed it); layer i > 0 gets the float64 chain's
    activation of layer i - 1 (the seeded network; x 4 for the random-weight variant)."""
    from bufferx_b200 import ops
    model, prep = c2["model"], c2["prep"]
    Kt = c2["delta"].shape[0]
    feat = ops.from_blocked(ops.spt_pnt(c2["delta"], prep["voxels"], prep["rot"], 0.8 / 3, 10, prep["w_pnt"], prep["b_pnt"], 20))
    L = model.Desc.conv_net.folded()
    t0 = time.perf_counter()
    _, aux = oracle.desc_fp64(feat, c2["sd"], keep=True)
    out = {}
    for name, layers, scale in (("seeded", L, 1.0), ("random", random_layers(L, dev), 4.0)):
        ins = [feat.view(Kt, 16, 3, 7, 20)] + [(a * scale).float() for a in aux["acts"][:7]]
        refs = [layer64(x.double(), l, i == 0) for i, (x, l) in enumerate(zip(ins, layers))]
        out[name] = dict(L=layers, ins=ins, refs=refs)
    torch.cuda.synchronize()
    out["t64"] = time.perf_counter() - t0
    out["acts"], out["feat"] = aux["acts"], feat
    return out


def run_layer(dev, route, i, l, x, K):
    """One layer on one route -> float [K, Cout, 140] (and the decoded padded raster for a presplit output)."""
    from bufferx_b200 import ops
    cout = l["cout"]
    first = i == 0
    geom = ops.GEOM_CYL3D if first else ops.GEOM_CYL2D
    xf = x.reshape(K, x.shape[1], -1)                    # [K,16,420] or [K,Cin,140]
    if route == "tf32":
        out = torch.full((K, cout // 4, 140, 4), float("nan"), device=dev)
        if first:
            ops.conv_layer_tc(geom, ops.to_blocked(xf), l["w_tc"], l["b"], out, K, 16, cout, 3, 7, 20, 3, 3, 3, l["relu"])
        else:
            ops.conv_layer_tc(geom, ops.to_blocked(xf), l["w_tc"], l["b"], out, K, l["cin"], cout, 1, 7, 20, 1, 3, 3, l["relu"])
        return ops.from_blocked(out), None
    if route == "fp32in":
        xin = ops.to_blocked(xf)
    else:
        xin = ops.sd_pack(x48(xf) if first else x.reshape(K, -1, 7, 20))
    presplit_out = route == "sd" and i < 7
    if presplit_out:
        out = nan_fp16((cout // 16, 4, ops.conv_sd_rows(K), 8), dev)
    else:
        out = torch.full((K, cout // 4, 140, 4), float("nan"), device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.conv_layer_sd(geom, xin, l["w_sd"], l["b"], out, K, l["cin"], cout, l["relu"], flag)
    assert int(flag.item()) == 0
    if presplit_out:
        val, xp = ops.sd_unpack(out, K)
        assert (xp[:, :, 0] == 0).all() and (out[:, :, K * 176:K * 176 + 22] == 0).all(), "zero rows of the presplit output"
        assert torch.equal(xp[:, :, 1:, 0], xp[:, :, 1:, 20]) and torch.equal(xp[:, :, 1:, 21], xp[:, :, 1:, 1]), "wrap columns"
        return val.reshape(K, cout, 140), xp
    return ops.from_blocked(out), None


@pytest.mark.parametrize("variant", ["seeded", "random"])
@pytest.mark.parametrize("K", [1, 2, 3, 37, 1500, 9000])
def test_cylindrical_layers_vs_fp64(dev, c2, chain, variant, K):
    """Every layer on every route against float64, elementwise.  sd: the production route (L0 reads the 3-chunk CYL3D
    presplit image -- the one bx_spt_pnt_sd writes, identical to sd_pack of the features -- L1-L6 presplit to presplit, L7
    presplit to fp32); fp32in: fp32 channel-blocked input (the debug route's first layer), fp32 output; tf32: bx_conv_layer_tc."""
    from bufferx_b200 import ops
    ch = chain[variant]
    worst = {}
    for i, l in enumerate(ch["L"]):
        x = ch["ins"][i][:K]
        ref, absref = (a[:K].reshape(K, l["cout"], 140) for a in ch["refs"][i])
        if i == 0 and variant == "seeded":
            img = spt_sd_into(c2["delta"][:K].contiguous(), c2["prep"], nan_fp16((3, 4, ops.conv_sd_rows(K), 8), dev))
            n = K * 176 + 22
            assert torch.equal(img[:, :, :n].view(torch.int16), ops.sd_pack(x48(x.reshape(K, 16, 420)))[:, :, :n].view(torch.int16))
        for route in ("sd", "fp32in", "tf32"):
            got, _ = run_layer(dev, route, i, l, x, K)
            r = check(f"{variant} L{i} {route} K={K}", got, ref, absref)
            worst[route] = max(worst.get(route, 0.0), r)
    report(f"layers {variant} K={K}: " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()) + "; max", max(worst.values()))


def test_cylindrical_net_chain_vs_fp64(dev, c2, chain):
    """All eight layers GPU to GPU at 9000 patches through Cylindrical_Net.forward on the three routes (presplit image from
    bx_spt_pnt_sd; fp32 features; TF32), against the float64 chain, elementwise: eight layers' worth of KAPPA times the last
    layer's absref on the float64 chain's own input.  (The first-order bound that pushes every layer's error on through |W|
    is no test here: with up to 1152 terms a layer it grows by ~10^11 over the stack.)"""
    from bufferx_b200 import ops
    net = c2["model"].Desc.conv_net
    Kt = c2["delta"].shape[0]
    feat = chain["feat"]
    ref = chain["acts"][7].reshape(Kt, 32, 140)
    a_abs = chain["seeded"]["refs"][7][1].reshape(Kt, 32, 140)
    img = ops.spt_pnt_sd(c2["delta"], c2["prep"]["voxels"], c2["prep"]["rot"], 0.8 / 3, 10, c2["prep"]["w_pnt"], c2["prep"]["b_pnt"], 20)
    msg = []
    with torch.no_grad():
        for route in ("sd", "fp32in", "tf32"):
            net.force_tf32 = route == "tf32"
            try:
                x, _ = net(img, K=Kt) if route == "sd" else net(ops.to_blocked(feat))
            finally:
                net.force_tf32 = False
            r = check(f"chain {route}", ops.from_blocked(x), ref, a_abs, kappa=8 * KAPPA)
            msg.append(f"{route} {r:.3g}")
    assert int(net.overflow_flag(dev).item()) == 0
    report(f"chain of eight layers, 9000 patches (float64 reference {chain['t64']:.2f} s on the GPU), err / absref of the last layer: " + ", ".join(msg)
           + "; max", max(float(m.split()[1]) for m in msg))


# ------------------------------------------------------------------------------------------------ 4. attention pooling
def pool64(x, prep):
    """bx_pool_desc in float64 on the folded pooling weights -> (desc, equi, pooled, absref of pooled, att)."""
    w1, b1 = prep["w1"].double(), prep["b1"].double()          # [32,16], [16]
    w2, b2 = prep["w2"].double(), prep["b2"].double()          # [16], [1]
    K = x.shape[0]
    xs = x.double().reshape(K, 32, 140)
    h = torch.einsum("kcs,cj->kjs", xs, w1) + b1.view(1, 16, 1)
    att = torch.relu(torch.einsum("kjs,j->ks", torch.relu(h), w2) + b2)
    pooled = (xs * att[:, None]).mean(dim=2)
    h_abs = torch.einsum("kcs,cj->kjs", xs.abs(), w1.abs()) + b1.abs().view(1, 16, 1)
    att_abs = torch.einsum("kjs,j->ks", h_abs, w2.abs()) + b2.abs()
    p_abs = (xs.abs() * att_abs[:, None]).mean(dim=2)
    nrm = pooled.norm(dim=1, keepdim=True)
    xn = xs.norm(dim=1, keepdim=True)
    return pooled / nrm.clamp(min=1e-12), xs / xn.clamp(min=1e-12), pooled, p_abs, att


def zero_attention_input(prep):
    """A position vector x [32] with relu(w2 . relu(W1^T x + b1) + b2) = 0, or None if the folded weights allow none."""
    w1, b1, w2, b2 = (prep[k].double().cpu() for k in ("w1", "b1", "w2", "b2"))
    neg = w2 < 0
    if float(b2) <= 0:
        t = -1.0 - b1.abs()                                   # every hidden unit off
    elif neg.any():
        j = int(torch.argmin(w2))
        t = -1.0 - b1.abs()
        t[j] = (float(b2) + 1.0) / float(-w2[j]) + 1.0        # one negative-weight unit carries w2 . h below -b2
    else:
        return None
    x = torch.linalg.lstsq(w1.t(), (t - b1).view(16, 1)).solution.view(32)
    return x.float()


def _pool_check(name, dev, oracle, sd, x, prep):
    """bx_pool_desc on x [K,32,7,20] with the folded pooling weights ``prep``, both input layouts (same bits), against
    float64: equi elementwise; desc within KAPPA * absref / |pooled| (the pooled vector carries KAPPA * absref, the
    normalisation divides by max(|pooled|, 1e-12) and adds at most |d| |KAPPA * absref| / |pooled|), or 1.5 x the fp32
    oracle's own error on that row.  -> (desc, equi, pooled, att, equi ratio, desc err / bound)."""
    from bufferx_b200 import ops
    K = x.shape[0]
    d64, e64, pooled, p_abs, att = pool64(x, prep)
    desc, equi = ops.pool_desc(x.contiguous(), prep["w1"], prep["b1"], prep["w2"], prep["b2"])
    d2, e2 = ops.pool_desc(ops.to_blocked(x.reshape(K, 32, 140)), prep["w1"], prep["b1"], prep["w2"], prep["b2"], channels_last=True)
    assert torch.equal(d2, desc) and torch.equal(e2, equi), f"{name}: the two input layouts differ"
    assert torch.isfinite(desc).all() and torch.isfinite(equi).all(), name
    re = check(f"{name} equi", equi.reshape(K, 32, 140), e64, e64.abs())
    nrm = pooled.norm(dim=1, keepdim=True).clamp(min=1e-12)
    bound = KAPPA * (p_abs + d64.abs() * p_abs.norm(dim=1, keepdim=True)) / nrm
    # the fp32 oracle on the same folded weights (the reference-keyed state_dict with the pooling layers replaced)
    W1, W2 = prep["w1"].t().reshape(16, 32, 1, 1).cpu(), prep["w2"].reshape(1, 16, 1, 1).cpu()
    sd1 = {"Desc.pool_layer.0.weight": W1, "Desc.pool_layer.0.bias": prep["b1"].cpu(),
           "Desc.pool_layer.3.weight": W2, "Desc.pool_layer.3.bias": prep["b2"].cpu()}
    for j, c in ((1, 16), (4, 1)):
        sd1.update({f"Desc.pool_layer.{j}.running_mean": torch.zeros(c), f"Desc.pool_layer.{j}.running_var": torch.full((c,), 1 - 1e-5),
                    f"Desc.pool_layer.{j}.weight": torch.ones(c), f"Desc.pool_layer.{j}.bias": torch.zeros(c)})
    with torch.no_grad():
        d32, _ = oracle.pool_desc(x.cpu(), sd1)
    e32 = (d32.double().to(dev) - d64).abs().max(dim=1, keepdim=True).values
    err = (desc.double() - d64).abs()
    bad = (err > bound) & (err > 1.5 * e32)
    assert not bad.any(), f"{name} desc: {int(bad.any(dim=1).sum())} rows beyond the bound"
    return desc, equi, pooled, att, re, float((err / bound.clamp(min=1e-300)).max())


def test_pool_desc_vs_fp64(dev, oracle, c2, chain):
    """bx_pool_desc on the chain's last activation (1500 patches) plus edge rows: a position with all 32 channels zero
    (equi 0, not NaN), an all-zero patch (desc 0), a patch whose attention is zero everywhere (desc 0); then pooled vectors
    of norm ~1e-9 and ~1e-13 (below the 1e-12 clamp), made by scaling the last attention layer by eps: relu(eps z) =
    eps relu(z), so the pooled vector scales by eps while x and its conditioning stay those of real patches."""
    prep = c2["prep"]
    K = 1500
    x = chain["acts"][7][:K].float().clone()                   # [K,32,7,20]
    x[0, :, 3, 5] = 0                                          # one position with all channels zero
    x[1] = 0                                                   # all-zero patch
    xz = zero_attention_input(prep)
    if xz is not None:
        x[2] = xz.to(dev).view(32, 1, 1) * (1 + 0.1 * torch.rand(1, 7, 20, device=dev))
    desc, equi, pooled, att, re, rd = _pool_check("pool", dev, oracle, c2["sd"], x, prep)
    assert (equi[0, :, 3, 5] == 0).all() and (equi[1] == 0).all() and (desc[1] == 0).all()
    if xz is not None:
        assert float(att[2].abs().max()) == 0 and (desc[2] == 0).all()
    pn = pooled.norm(dim=1)
    msg = [f"{int((pn[3:] == 0).sum())} of {K - 3} real patches have zero attention everywhere (desc 0)"]
    rows = torch.argsort(pn, descending=True)[:32]             # the best-conditioned real rows
    ref_n = float(pn[rows].min())
    for target in (1e-9, 1e-13):
        eps = target / ref_n
        pe = dict(prep, w2=(prep["w2"].double() * eps).float(), b2=(prep["b2"].double() * eps).float())
        _, _, pooled_e, _, r_e, rd_e = _pool_check(f"pool |pooled| ~ {target:g}", dev, oracle, c2["sd"], x[rows], pe)
        re, rd = max(re, r_e), max(rd, rd_e)
        msg.append(f"|pooled| {float(pooled_e.norm(dim=1).min()):.3g}..{float(pooled_e.norm(dim=1).max()):.3g}: desc err / bound {rd_e:.3g}")
    print("\n[descnet-fp64] pool edge rows: " + "; ".join(msg) + f"; zero-attention row {'built' if xz is not None else 'impossible'}")
    report("pool_desc: equi ratio", re)
    report("pool_desc: desc err / bound", rd)


# ------------------------------------------------------------------------------------------------ 5+6. whole route
def rel_rows(a, b):
    den = b.abs().amax(dim=1)
    return (a - b).abs().amax(dim=1) / torch.where(den > 0, den, torch.ones_like(den))


def fp32_oracle_desc(oracle, inv, sd, dev):
    """The fp32 oracle (pnt_max -> cyl_net -> pool_desc) run through torch fp32 on the GPU with TF32 off."""
    sd = {k: v.to(dev) for k, v in sd.items() if k.startswith("Desc.")}
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            out = []
            for s in range(0, inv.shape[0], 1500):
                f = oracle.pnt_max(torch.from_numpy(inv[s:s + 1500]).to(dev), sd)
                x = oracle.cyl_net(f.view(f.shape[0], 16, 3, 7, 20), sd)
                out.append(oracle.pool_desc(x, sd)[0])
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    return torch.cat(out).double()


def compare_rows(name, d, d64, d32):
    """The per-row rule of test_gpu_parity._compare_pair on every row: wherever the GPU and the fp32 oracle disagree beyond
    1e-4, the GPU is within 1.5 x the oracle's own error from float64 (+ 2e-5); everywhere else within 1e-4 of float64."""
    d = d.double()
    rel = rel_rows(d, d32)
    e_gpu, e_orc = rel_rows(d, d64), rel_rows(d32, d64)
    off = rel >= 1e-4
    bad = off & (e_gpu > 1.5 * e_orc + 2e-5)
    assert not bad.any(), f"{name}: GPU vs fp64 {e_gpu[bad][:5].tolist()} against oracle vs fp64 {e_orc[bad][:5].tolist()}"
    assert (e_gpu[~off] < 1e-4).all(), f"{name}: GPU vs fp64 {float(e_gpu[~off].max())}"
    assert float(e_gpu.median()) < 2e-5
    return (f"{name}: {len(d)} rows, GPU vs float64 max {float(e_gpu.max()):.3g} median {float(e_gpu.median()):.3g}, "
            f"fp32 oracle vs float64 max {float(e_orc.max()):.3g}, {int(off.sum())} rows where GPU and oracle differ by >= 1e-4")


def test_forward_multi_c2_pair_every_row_vs_fp64(dev, oracle, c2):
    """The production route at production size: forward_multi's 9000 descriptors of the C2 pair, every row, against
    oracle.desc_fp64 of the float64 point-layer features."""
    t0 = time.perf_counter()
    d64 = oracle.desc_fp64(c2["feat64"], c2["sd"])
    torch.cuda.synchronize()
    t64 = time.perf_counter() - t0
    d32 = fp32_oracle_desc(oracle, c2["einv"], c2["sd"], dev)
    msg = compare_rows("forward_multi C2", c2["desc"], d64, d32)
    print(f"\n[descnet-fp64] {msg}; float64 reference {t64:.2f} s on the GPU")


def test_fp16_overflow_switches_to_tf32_end_to_end(dev, oracle, c2):
    """The point layer scaled so that the pair's features pass 65000: forward() on the production route raises the
    fp16-range flag, switches to the TF32 kernels by itself and recomputes the pair; its descriptors meet the per-row rule
    against float64 of the scaled network."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights
    s = 1.2e5 / float(c2["feat64"].max())
    sd = {k: v.clone() for k, v in c2["sd"].items()}
    for k in ("pnt_layer.0.weight", "pnt_layer.0.bias", "pnt_layer.1.running_mean", "pnt_layer.1.bias"):
        sd["Desc." + k] = sd["Desc." + k] * s            # BN(s conv(x)) with s-scaled mean and shift = s BN(conv(x))
    model = init_synthetic_weights(bx.BufferX(c2["cfg"]), trained_pose=True)
    model.load_state_dict(sd)
    model = model.to(dev).eval()
    with torch.no_grad():
        model(c2["data"], perms=c2["perms"], ransac_seed=0)
    assert model.Desc.conv_net.force_tf32 and model.Pose.conv.force_tf32, "the fp16-range flag did not switch to TF32"
    assert int(model.Desc.conv_net.overflow_flag(dev).item()) == 0
    desc = model.Desc.last_multi["desc"].clone()
    feat64 = oracle.pnt_fp64(c2["delta"], c2["evidx"], sd)
    assert float(feat64.max()) > 65000
    d64 = oracle.desc_fp64(feat64, sd)
    d32 = fp32_oracle_desc(oracle, c2["einv"], sd, dev)
    msg = compare_rows("overflow -> TF32", desc, d64, d32)
    print(f"\n[descnet-fp64] {msg}; largest feature {float(feat64.max()):.3g}")
