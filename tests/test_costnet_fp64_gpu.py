"""CostNet (a11) and the hypothesis build (a12) on the GPU against float64, layer by layer.

Each kernel is compared elementwise with the same operation evaluated in float64 on the same fp32 inputs:
|got - ref| <= KAPPA * absref, where absref is that layer in float64 with |x|, |W| and |b|, so a small output cannot hide
behind a max-normalised error.  KAPPA = 2e-5: the fp16 hi/lo split keeps about 2^-22 of each product, and the fp32 running
sums are folded per 16-channel chunk of 144 products (144 * 2^-24 ~ 9e-6 at worst).  The largest ratio of each test is
printed (run with -s) and recorded in DESIGN.md section 7."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

KAPPA = 2e-5


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def nets(dev):
    """The fitted and the seeded random CostNet: model on the GPU, reference-keyed state_dict on the host."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    out = {}
    for name, fitted in (("fitted", True), ("random", False)):
        model = init_synthetic_weights(bx.BufferX(workload_cfg("C2")), trained_pose=fitted)
        sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
        out[name] = dict(model=model.to(dev).eval(), sd=sd)
    return out


def report(name, value):
    print(f"\n[costnet-fp64] {name}: {value:.3g}")


# ------------------------------------------------------------------------------------------------ inputs
def equi_maps(K, kind, seed):
    """Equivariant maps (es, et) [K,32,7,20] fp32.  prod: L2-normalised over channels, as pool_desc writes them; et[j] is
    es[j] rolled by a random integer azimuth plus 1e-3 noise for j < K / 2 (a match list pairing j with j then hits a cost
    volume that is ~0 at one n), independent for the rest.  raw: randn * 4, not normalised."""
    g = torch.Generator().manual_seed(seed)
    if kind == "raw":
        return 4 * torch.randn(K, 32, 7, 20, generator=g), 4 * torch.randn(K, 32, 7, 20, generator=g)
    es = F.normalize(torch.randn(K, 32, 7, 20, generator=g), dim=1)
    et = F.normalize(torch.randn(K, 32, 7, 20, generator=g), dim=1)
    shifts = torch.randint(0, 20, (K,), generator=g)
    for j in range(K // 2):
        et[j] = F.normalize(torch.roll(es[j], int(shifts[j]), dims=2) + 1e-3 * torch.randn(32, 7, 20, generator=g), dim=0)
    return es, et


def match_lists(K, maxM, seed):
    """int32 (s_mids, t_mids) [maxM]: repeated indices, indices 0 and K - 1, non-monotone t, and pairs (j, j) with j < K / 2."""
    rng = np.random.default_rng(seed)
    s = rng.integers(0, K, maxM)
    t = rng.integers(0, K, maxM)
    true = rng.random(maxM) < 0.5
    s[true] = rng.integers(0, max(K // 2, 1), int(true.sum()))
    t[true] = s[true]
    s[0], t[0] = 0, K - 1
    if maxM > 1:
        s[1], t[1] = K - 1, 0
    if maxM > 3:
        s[3], t[3] = s[2], t[2]
    return torch.from_numpy(s.astype(np.int32)), torch.from_numpy(t.astype(np.int32))


# ------------------------------------------------------------------------------------------------ float64 references
def w5(Wt, k):
    """Folded [T, Cin, Cout] -> float64 conv weight [Cout, Cin, *k]."""
    return Wt.detach().cpu().double().permute(2, 1, 0).reshape(Wt.shape[2], Wt.shape[1], *k)


def layer64(x, L, relu=True):
    """(out, absref) of one folded layer in float64: x [M, Cin, D, H, W]."""
    W, b = w5(L["w"], L["k"]), L["b"].detach().cpu().double()
    out = F.conv3d(x, W, b)
    return (torch.relu(out) if relu else out), F.conv3d(x.abs(), W.abs(), b.abs())


def factors64(d1, d2, wa, wb, bias):
    """A [M,32,3,20], B [M,32,3,18] of bx_costvol_ab in float64 (maps [M,32,5,20]) and their absref."""
    def circ(x):
        return torch.cat([x[..., -2:], x, x[..., :2]], dim=-1)          # column j -> azimuth (j - 2) mod 20
    Wa, Wb, b = wa.cpu().double().permute(3, 0, 1, 2), wb.cpu().double().permute(3, 0, 1, 2), bias.cpu().double().view(1, -1, 1, 1)
    x1, x2 = circ(d1.double()), d2.double()
    return F.conv2d(x1, Wa) + b, F.conv2d(x2, Wb), F.conv2d(x1.abs(), Wa.abs()) + b.abs(), F.conv2d(x2.abs(), Wb.abs())


def cost_parts(d1, d2):
    """The two halves of the cost volume [M,C,n,k,l]: d1[c,k,(l-n) mod 20] and d2[c,k,l] (oracle.cost_volume)."""
    M, C, H, _ = d1.shape
    l = torch.arange(20)
    idx = (l[None, :] - l[:, None]) % 20
    v1 = d1[:, :, :, idx.reshape(-1)].reshape(M, C, H, 20, 20).permute(0, 1, 3, 2, 4)
    return v1, d2.unsqueeze(2).expand(M, C, 20, H, 20)


def regenerate(A, B):
    """relu(A[c,k,(l-n) mod 20] - B[c,k,l]) -> [M,32,18(n),3(k),18(l)]."""
    n = torch.arange(18).view(18, 1)
    l = torch.arange(18).view(1, 18)
    return torch.relu(A[:, :, :, (l - n) % 20] - B[:, :, :, None, :]).permute(0, 1, 3, 2, 4)


def gather(e, idx):
    """Elevation rows 1..5 of the maps of a match list -> [M,32,5,20]."""
    return e[idx.long()][:, :, 1:6]


# ------------------------------------------------------------------------------------------------ presplit valid rasters
def valid_pack(x, dev):
    """[n, C, D, W] (rows of NaN allowed) -> the presplit image [C/16, 4, rows, 8] fp16 of a valid raster of D * W rows per
    sample (bx_conv_layer_sd VALID3D input): x = hi + lo * 2^-11, zero halo rows."""
    from bufferx_b200 import ops
    n, C, D, W = x.shape
    rows = ops.conv_sd_rows(n, D * W)
    flat = torch.zeros((rows, C), dtype=torch.float32)
    flat[: n * D * W] = x.float().permute(0, 2, 3, 1).reshape(n * D * W, C)
    hi = flat.half()
    lo = ((flat - hi.float()) * 2048.0).half()
    img = torch.stack([hi, lo], dim=0).view(2, rows, C // 16, 2, 8).permute(2, 0, 3, 1, 4).contiguous()   # [chunk, split, kcore, rows, 8]
    return img.view(C // 16, 4, rows, 8).to(dev)


def valid_unpack(img, n, D, W):
    """Presplit image of a valid raster -> float64 [n, C, D, W] (hi + lo * 2^-11)."""
    nch, _, rows, _ = img.shape
    v = img.detach().cpu().view(nch, 2, 2, rows, 8).double()
    flat = (v[:, 0] + v[:, 1] / 2048.0).permute(2, 0, 1, 3).reshape(rows, nch * 16)
    return flat[: n * D * W].view(n, D, W, nch * 16).permute(0, 3, 1, 2)


def nan_fp16(shape, dev):
    return torch.full(shape, float("nan"), dtype=torch.float16, device=dev)


def check(name, got, ref, absref, kappa=KAPPA):
    """Elementwise |got - ref| <= kappa * absref (both float64, same shape); returns the largest ratio."""
    err = (got.double() - ref).abs()
    ratio = float((err / absref.clamp(min=1e-30)).max())
    bad = err > kappa * absref
    assert not bad.any(), f"{name}: {int(bad.sum())} elements beyond {kappa} * absref, worst ratio {ratio:.3g}"
    assert torch.isfinite(got).all(), name
    return ratio


# ------------------------------------------------------------------------------------------------ G1 bx_costvol_ab
@pytest.mark.parametrize("net", ["fitted", "random"])
@pytest.mark.parametrize("kind", ["prod", "raw"])
def test_costvol_ab_vs_fp64(dev, nets, net, kind):
    """A and B against float64 from the same fp32 maps and factor weights; relu(A - B) against the direct first layer
    (cost volume -> conv); rows >= d_M keep their NaN sentinel and d_M = 0 writes nothing."""
    from bufferx_b200 import ops
    L0 = nets[net]["model"].Pose.conv.folded()[0]
    wa, wb = ops.costvol_factor_weights(L0["w"])
    K, maxM, dM = 300, 260, 250
    es, et = equi_maps(K, kind, 11)
    sm, tm = match_lists(K, maxM, 12)
    A = torch.full((maxM, 8, 60, 4), float("nan"), device=dev)
    B = torch.full((maxM, 8, 54, 4), float("nan"), device=dev)
    ops.costvol_ab(es.to(dev), et.to(dev), sm.to(dev), tm.to(dev), torch.tensor([dM], dtype=torch.int32, device=dev), maxM,
                   wa, wb, L0["b"], A, B)
    assert torch.isnan(A[dM:]).all() and torch.isnan(B[dM:]).all()
    Ag = ops.from_blocked(A[:dM]).view(dM, 32, 3, 20).cpu().double()
    Bg = ops.from_blocked(B[:dM]).view(dM, 32, 3, 18).cpu().double()
    d1, d2 = gather(es, sm[:dM]), gather(et, tm[:dM])
    A64, B64, absA, absB = factors64(d1, d2, wa, wb, L0["b"])
    ra = check("A", Ag, A64, absA)
    rb = check("B", Bg, B64, absB)
    # the factorised first activation against the direct layer on a strided subset of the matches
    sub = torch.arange(0, dM, 5)
    v1, v2 = cost_parts(d1[sub].double(), d2[sub].double())
    W = w5(L0["w"], (3, 3, 3))
    b = L0["b"].cpu().double()
    ref = torch.relu(F.conv3d(v1 - v2, W, b))
    absref = F.conv3d(v1.abs(), W.abs()) + F.conv3d(v2.abs(), W.abs()) + b.abs().view(1, -1, 1, 1, 1)
    r0 = check("relu(A - B)", regenerate(Ag[sub], Bg[sub]), ref, absref)
    report(f"G1 costvol_ab {net}/{kind}: A, B, relu(A - B)", max(ra, rb, r0))
    # d_M = 0: nothing is written
    A.fill_(float("nan")); B.fill_(float("nan"))
    ops.costvol_ab(es.to(dev), et.to(dev), sm.to(dev), tm.to(dev), torch.zeros(1, dtype=torch.int32, device=dev), maxM,
                   wa, wb, L0["b"], A, B)
    assert torch.isnan(A).all() and torch.isnan(B).all()


# ------------------------------------------------------------------------------------------------ G2 bx_conv_layer_sd_costab
def _costab_factors(dev, nets, maxM, kind):
    """fp32 factor maps (A, B) channel-blocked [maxM,8,60,4] / [maxM,8,54,4]: from bx_costvol_ab on production-like maps, or
    arbitrary values."""
    from bufferx_b200 import ops
    if kind == "arbitrary":
        g = torch.Generator().manual_seed(maxM)
        return (torch.randn(maxM, 8, 60, 4, generator=g).to(dev), torch.randn(maxM, 8, 54, 4, generator=g).to(dev))
    L0 = nets["fitted"]["model"].Pose.conv.folded()[0]
    wa, wb = ops.costvol_factor_weights(L0["w"])
    K = max(maxM, 8)
    es, et = equi_maps(K, "prod", 21)
    sm, tm = match_lists(K, maxM, 22)
    return ops.costvol_ab(es.to(dev), et.to(dev), sm.to(dev), tm.to(dev), torch.tensor([maxM], dtype=torch.int32, device=dev),
                          maxM, wa, wb, L0["b"])


@pytest.mark.parametrize("maxM", [1, 2, 3, 37, 1500])
def test_costab_layer_vs_fp64(dev, nets, maxM):
    """The second CostNet layer (relu(A - B) regenerated in the loader, 96 -> 64 over the 18 x 18 raster) against the float64
    3x3x3 conv over relu(A - B) built from the same fp32 factors.  324-row samples straddle 128-row tiles; at 1500 samples
    the persistent CTAs loop over 3797 tiles.  fp32 and presplit output, rows of samples >= d_M untouched.  The same layer on
    the TF32 kernel (bx_conv_layer_tc, GEOM_COSTAB: the fp16-range fall-back) is held to the same bound."""
    from bufferx_b200 import ops
    L1 = nets["fitted"]["model"].Pose.conv.folded()[1]
    w_sd = ops.conv_sd_weights_costab(L1["w"])

    def tf32(fa, fb, d_n, relu):
        out = torch.full((maxM, 16, 256, 4), float("nan"), device=dev)
        ops.conv_layer_tc(ops.GEOM_COSTAB, None, L1["w_tc"], L1["b"], out, maxM, 32, 64, 18, 3, 18, 3, 3, 3, relu, d_n=d_n,
                          equi_s=fa, equi_t=fb)
        return ops.from_blocked(out).cpu()

    # at 1500 samples the float64 reference covers every 7th sample (7 is prime to the 32 tile phases of a 324-row sample)
    sub = torch.arange(maxM) if maxM < 100 else torch.cat([torch.arange(0, maxM, 7), torch.arange(maxM - 3, maxM)]).unique()
    worst = {"sd": 0.0, "tf32": 0.0}
    for kind in ("costvol_ab", "arbitrary"):
        fa, fb = _costab_factors(dev, nets, maxM, kind)
        A = ops.from_blocked(fa).view(maxM, 32, 3, 20).cpu().double()
        B = ops.from_blocked(fb).view(maxM, 32, 3, 18).cpu().double()
        x = regenerate(A[sub], B[sub])
        ref, absref = layer64(x, L1)                                           # [m, 64, 16, 1, 16]
        ref, absref = ref.view(-1, 64, 256), absref.view(-1, 64, 256)
        for dM in sorted({maxM, maxM - 1, 1, min(5, maxM), 0}):
            d_n = torch.tensor([dM], dtype=torch.int32, device=dev)
            live = sub < dM
            out = torch.full((maxM, 16, 256, 4), float("nan"), device=dev)
            ops.conv_layer_sd_costab(fa, fb, w_sd, L1["b"], out, maxM, True, d_n=d_n)
            got = ops.from_blocked(out).cpu()
            assert torch.isnan(got[dM:]).all(), f"fp32 rows of samples >= d_M = {dM} written"
            if dM:
                worst["sd"] = max(worst["sd"], check(f"costab fp32 {kind} d_M={dM}", got[sub[live]], ref[live], absref[live]))
            img = nan_fp16(ops.conv_sd_buffer(maxM, 64, dev, 256).shape, dev)
            ops.conv_layer_sd_costab(fa, fb, w_sd, L1["b"], img, maxM, True, d_n=d_n)
            assert torch.isnan(img[:, :, dM * 256:]).all(), f"presplit rows of samples >= d_M = {dM} written"
            if dM:
                dec = valid_unpack(img, maxM, 16, 16).reshape(maxM, 64, 256)
                worst["sd"] = max(worst["sd"], check(f"costab presplit {kind} d_M={dM}", dec[sub[live]], ref[live], absref[live]))
            got = tf32(fa, fb, d_n, True)
            assert torch.isnan(got[dM:]).all(), f"tf32 rows of samples >= d_M = {dM} written"
            if dM:
                worst["tf32"] = max(worst["tf32"], check(f"costab tf32 {kind} d_M={dM}", got[sub[live]], ref[live], absref[live]))
        if maxM == 37:                  # relu = False once
            pre, absref = layer64(x, L1, relu=False)
            out = torch.full((maxM, 16, 256, 4), float("nan"), device=dev)
            ops.conv_layer_sd_costab(fa, fb, w_sd, L1["b"], out, maxM, False, d_n=torch.tensor([maxM], dtype=torch.int32, device=dev))
            got = ops.from_blocked(out).cpu()
            assert (got < 0).any()
            worst["sd"] = max(worst["sd"], check(f"costab relu=False {kind}", got, pre.view(-1, 64, 256), absref.view(-1, 64, 256)))
            got = tf32(fa, fb, torch.tensor([maxM], dtype=torch.int32, device=dev), False)
            assert (got < 0).any()
            worst["tf32"] = max(worst["tf32"], check(f"costab tf32 relu=False {kind}", got, pre.view(-1, 64, 256), absref.view(-1, 64, 256)))
    report(f"G2 costab maxM={maxM}: sd {worst['sd']:.3g}, tf32 {worst['tf32']:.3g}; max", max(worst.values()))


@pytest.mark.parametrize("value,flagged", [(6e4, 0), (7e4, 1)])
def test_costab_fp16_range_flag(dev, nets, value, flagged):
    """The loader raises the fp16-range flag when a regenerated activation reaches 65000."""
    from bufferx_b200 import ops
    L1 = nets["fitted"]["model"].Pose.conv.folded()[1]
    n = 4
    fa = torch.zeros((n, 8, 60, 4), device=dev)
    fb = torch.zeros((n, 8, 54, 4), device=dev)
    fa[2, 3, 25, 1] = value                           # channel 13, (k = 1, m = 5) of sample 2
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    out = torch.empty((n, 16, 256, 4), device=dev)
    ops.conv_layer_sd_costab(fa, fb, ops.conv_sd_weights_costab(L1["w"]), L1["b"], out, n, True, flag,
                             d_n=torch.tensor([n], dtype=torch.int32, device=dev))
    assert int(flag.item()) == flagged


# ------------------------------------------------------------------------------------------------ G3 the k = (3,1,3) layers
@pytest.mark.parametrize("net", ["fitted", "random"])
def test_valid_layers_vs_fp64(dev, nets, oracle, net):
    """The seven k = (3,1,3) layers in production order (16 x 16 -> 14 -> ... -> 2; 64 -> 64 -> 128 -> 128 -> 64 -> 64 ->
    32 -> 32).  Each layer gets the float64 chain's previous activation packed as presplit input and is bounded per layer;
    then the whole chain runs GPU to GPU with presplit hand-off and is bounded against the float64 chain."""
    from bufferx_b200 import ops
    model, sd = nets[net]["model"], nets[net]["sd"]
    L = model.Pose.conv.folded()
    K, maxM, dM = 120, 45, 43                          # the 4 x 4 raster: 16 rows a sample, 8 samples a tile, 10 halo rows
    es, et = equi_maps(K, "prod", 31)
    sm, tm = match_lists(K, maxM, 32)
    _, acts = oracle.costnet_fp64(gather(es, sm[:dM]), gather(et, tm[:dM]), sd, keep=True)
    d_n = torch.tensor([dM], dtype=torch.int32, device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)

    def padded(a):              # [dM, C, D, 1, W] -> [maxM, C, D, W] with NaN for the samples past d_M
        x = torch.full((maxM,) + tuple(a.shape[1:3]) + (a.shape[4],), float("nan"), dtype=torch.float64)
        x[:dM] = a[:, :, :, 0]
        return x

    worst = {}
    D = 16
    for i in range(2, 9):
        l = L[i]
        assert l["k"] == (3, 1, 3) and l["w_sd"] is not None
        x = acts[i - 1]
        ref, absref = layer64(x, l)
        OD = D - 2
        out = torch.full((maxM, l["cout"] // 4, OD * OD, 4), float("nan"), device=dev)
        ops.conv_layer_sd(ops.GEOM_VALID3D, valid_pack(padded(x), dev), l["w_sd"], l["b"], out, maxM, l["cin"], l["cout"], True,
                          flag, d_n=d_n, D=D, W=D)
        got = ops.from_blocked(out).cpu()
        assert torch.isnan(got[dM:]).all()
        worst[i] = check(f"layer {i} ({l['cin']}->{l['cout']}, {D}x{D})", got[:dM], ref.reshape(dM, l["cout"], -1),
                         absref.reshape(dM, l["cout"], -1))
        D = OD
    # GPU to GPU: layer 1's float64 activation in, presplit between the layers, fp32 out of the last one
    cur, D = valid_pack(padded(acts[1]), dev), 16
    a_abs = acts[1].abs()
    for i in range(2, 9):
        l = L[i]
        OD = D - 2
        last = i == 8
        out = (torch.full((maxM, l["cout"] // 4, OD * OD, 4), float("nan"), device=dev) if last
               else ops.conv_sd_buffer(maxM, l["cout"], dev, OD * OD))
        ops.conv_layer_sd(ops.GEOM_VALID3D, cur, l["w_sd"], l["b"], out, maxM, l["cin"], l["cout"], True, flag, d_n=d_n, D=D, W=D)
        a_abs = F.conv3d(a_abs, w5(l["w"], l["k"]).abs(), l["b"].cpu().double().abs())     # the chain in |x|, |W|, |b|
        cur, D = out, OD
    got = ops.from_blocked(cur).cpu()
    assert torch.isnan(got[dM:]).all()
    # a forward error bound: each of the seven layers adds KAPPA * absref and passes on the earlier errors through |W|
    worst["chain"] = check("chain", got[:dM], acts[8].reshape(dM, 32, 4), a_abs.reshape(dM, 32, 4), kappa=8 * KAPPA) / 8
    assert int(flag.item()) == 0
    report(f"G3 k=(3,1,3) layers {net}: per layer " + ", ".join(f"{k}: {v:.3g}" for k, v in worst.items()) + "; max",
           max(worst.values()))


# ------------------------------------------------------------------------------------------------ G4 whole CostNet, every route
def _case(name, dev, c2_runs):
    """(equi_s, equi_t, s_mids, t_mids, d_M tensor, maxM, reference rows) on the GPU."""
    from bufferx_b200 import ops
    if name == "c1":
        es, et = equi_maps(256, "prod", 41)
        sm, tm = match_lists(256, 256, 42)
        return es.to(dev), et.to(dev), sm.to(dev), tm.to(dev), 200, 256, torch.arange(200)
    if name == "scale":
        es, et = equi_maps(1500, "prod", 43)
        sm, tm = match_lists(1500, 1500, 44)
        return es.to(dev), et.to(dev), sm.to(dev), tm.to(dev), 1300, 1500, torch.arange(1300)
    # the batched multi-scale path: three scales of a C2 pair, concatenated on the device (models/BUFFERX.py:375-378)
    run = c2_runs(0)
    K = run["cfg"].patch.num_fps
    scales = run["res"][5]["scales"]
    S = len(scales)
    equi = torch.cat([t for sc in scales for t in (sc["src"]["equi"], sc["tgt"]["equi"])]).contiguous().to(dev)
    s_lists = torch.zeros((S, K), dtype=torch.int32)
    t_lists = torch.zeros((S, K), dtype=torch.int32)
    cnts = torch.zeros(S, dtype=torch.int32)
    for i, sc in enumerate(scales):
        m = len(sc["s_mids"])
        s_lists[i, :m] = torch.from_numpy(sc["s_mids"].astype(np.int32))
        t_lists[i, :m] = torch.from_numpy(sc["t_mids"].astype(np.int32))
        cnts[i] = m
    offs = torch.zeros(S + 1, dtype=torch.int32, device=dev)
    s_all, t_all = ops.concat_matches(s_lists.to(dev), t_lists.to(dev), cnts.to(dev), [2 * i * K for i in range(S)],
                                      [(2 * i + 1) * K for i in range(S)], offs)
    total = int(cnts.sum())
    assert int(offs[S].item()) == total
    return equi, equi, s_all, t_all, total, S * K, torch.arange(0, total, 3)


def _logits(model, es, et, sm, tm, dM, maxM):
    with torch.no_grad():
        out = model.Pose.logits(es, et, sm, tm, torch.tensor([dM], dtype=torch.int32, device=es.device), maxM)
    torch.cuda.synchronize()
    return out.detach().cpu().clone()


@pytest.mark.parametrize("case,net", [("c1", "fitted"), ("c1", "random"), ("scale", "fitted"), ("batched", "fitted")])
def test_forward_matches_every_route_vs_fp64(dev, nets, oracle, c2_runs, monkeypatch, case, net):
    """CostNet.forward_matches on every route against oracle.costnet_fp64: per row, the GPU logit error is at most 1.5 x the
    fp32 oracle's + 2e-5 * max|logit|, and the soft arg-max bin is within 1e-4 of the float64 one.  The dynamic tile
    schedule gives the same bits as the static one."""
    from bufferx_b200 import ops
    from bufferx_b200.models import patchnet
    model, sd = nets[net]["model"], nets[net]["sd"]
    es, et, sm, tm, dM, maxM, rows = _case(case, dev, c2_runs)
    smh, tmh = sm[:dM].cpu()[rows], tm[:dM].cpu()[rows]
    d1, d2 = gather(es.cpu(), smh), gather(et.cpu(), tmh)
    l64 = oracle.costnet_fp64(d1, d2, sd)
    with torch.no_grad():
        l32, _ = oracle._cost_net(d1, d2, sd, 20, "Pose.conv.")
    err32 = (l32.double() - l64).abs().max(dim=1).values
    bound = 1.5 * err32 + 2e-5 * l64.abs().max(dim=1).values
    ind64 = oracle.soft_argmax(l64)
    # soft arg-max: 1e-4 (about 10x the fp32 oracle's error on a single peak).  d ind / d logit_k = p_k (k - ind), so a row
    # whose mass sits at both ends of the bin range turns the same fp32-grade logit error into a larger bin error: the bound
    # scales with s = sum p_k |k - ind| (<= 1 on a single peak) and is at least 1.5 x the fp32 oracle's own error; never
    # beyond 2e-4
    ind32_err = (oracle.soft_argmax(l32) - ind64).abs()
    p = torch.softmax(l64, dim=1)
    s = (p * (torch.arange(20, dtype=torch.float64)[None] - ind64[:, None]).abs()).sum(dim=1)
    ind_bound = torch.clamp(torch.maximum(1e-4 * s.clamp(min=1.0), 1.5 * ind32_err), max=2e-4)

    def worst_row(dind):
        r = int((dind - ind_bound).argmax())
        return (f"{float(dind.max()):.3g} from float64; worst row vs its bound: err {float(dind[r]):.3g}, s {float(s[r]):.3g}, "
                f"fp32 oracle {float(ind32_err[r]):.3g}")

    conv = model.Pose.conv
    routes = {}
    routes["default"] = _logits(model, es, et, sm, tm, dM, maxM)
    conv.force_tf32 = True
    try:
        routes["tf32"] = _logits(model, es, et, sm, tm, dM, maxM)
    finally:
        conv.force_tf32 = False
    monkeypatch.setattr(patchnet, "DYNAMIC_TILES", True)
    routes["dynamic"] = _logits(model, es, et, sm, tm, dM, maxM)
    monkeypatch.undo()
    assert torch.equal(routes["dynamic"][:dM], routes["default"][:dM]), "dynamic tiles changed the logits"
    msg = []
    for name, lg in routes.items():
        got = lg[:dM][rows].double()
        err = (got - l64).abs().max(dim=1).values
        bad = err > bound
        assert not bad.any(), f"{name}: {int(bad.sum())} rows beyond 1.5 x oracle error + 2e-5 max|logit|, worst {float((err - bound).max()):.3g}"
        dind = (oracle.soft_argmax(got) - ind64).abs()
        assert (dind <= ind_bound).all(), f"{name}: soft arg-max {worst_row(dind)}"
        msg.append(f"{name}: logit err / bound {float((err / bound).max()):.3g}, max logit err {float(err.max()):.3g}, "
                   f"soft arg-max {float(dind.max()):.3g} ({int((dind > 1e-4).sum())} rows > 1e-4)")
    msg.append(f"fp32 oracle: max logit err {float(err32.max()):.3g}, soft arg-max {float(ind32_err.max()):.3g} "
               f"({int((ind32_err > 1e-4).sum())} rows > 1e-4)")
    # the production soft arg-max: bx_hypotheses on the default route's logits
    ind = _hypotheses(dev, routes["default"].to(dev), dM, maxM)
    dind = (ind[:dM][rows].double() - ind64).abs()
    assert (dind <= ind_bound).all(), f"bx_hypotheses soft arg-max {worst_row(dind)}"
    msg.append(f"bx_hypotheses soft arg-max {float(dind.max()):.3g}")
    report(f"G4 {case}/{net} (M = {dM}, {len(rows)} rows checked): " + "; ".join(msg) + "; worst soft arg-max", float(dind.max()))


def _hypotheses(dev, logits, dM, maxM):
    """bx_hypotheses on logits with identity key-points / frames -> ind [maxM] (host)."""
    from bufferx_b200 import ops
    kp = torch.zeros((maxM, 3), device=dev)
    Rt = torch.eye(3, device=dev).expand(maxM, 3, 3).contiguous()
    ids = torch.arange(maxM, dtype=torch.int32, device=dev)
    offs = torch.zeros(2, dtype=torch.int32, device=dev)
    ind = torch.full((maxM,), float("nan"), device=dev)
    acc = [torch.empty((maxM, 3, 3), device=dev)] + [torch.empty((maxM, 3), device=dev) for _ in range(3)]
    ops.hypotheses(logits, 20, kp, kp, Rt, Rt, ids, ids, torch.tensor([dM], dtype=torch.int32, device=dev), maxM,
                   offs[0:1], offs[1:2], ind, *acc)
    return ind.cpu()


# ------------------------------------------------------------------------------------------------ G5 bx_hypotheses
def _rotations(n, rng):
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                     2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                     2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], axis=1).reshape(n, 3, 3)


def test_hypotheses_vs_fp64(dev, oracle):
    """Soft arg-max and pose hypotheses against the float64 formula: flat logits (9.5), one-hot at bin 0 (ind ~ 0: the Taylor
    branch of the rotation) and at 19, equal peaks at 0 and 19 (the expectation is not circular: 9.5), magnitudes of 80;
    appended at a non-zero row offset with every other accumulator row untouched."""
    from bufferx_b200 import ops
    rng = np.random.default_rng(51)
    rows = [np.zeros(20), np.eye(20)[0] * 80, np.eye(20)[19] * 80, np.eye(20)[0] * 30 + np.eye(20)[19] * 30,
            np.eye(20)[0] * 80 - 40, -80 * np.eye(20)[7], np.eye(20)[3] * 2.0]
    rows += list(rng.uniform(-80, 80, (20, 20))) + list(rng.normal(size=(80, 20)) * 3)
    logits = np.asarray(rows, dtype=np.float32)
    M, maxM, K, off = len(logits), len(logits) + 9, 64, 7
    kps, kpt = rng.uniform(-3, 3, (K, 3)).astype(np.float32), rng.uniform(-3, 3, (K, 3)).astype(np.float32)
    Rs, Rt = _rotations(K, rng).astype(np.float32), _rotations(K, rng).astype(np.float32)
    sm, tm = rng.integers(0, K, maxM).astype(np.int32), rng.integers(0, K, maxM).astype(np.int32)
    lg = torch.full((maxM, 20), float("nan"))
    lg[:M] = torch.from_numpy(logits)
    cap = off + maxM + 5
    R_acc = torch.full((cap, 3, 3), float("nan"), device=dev)
    t_acc, ss_acc, tt_acc = (torch.full((cap, 3), float("nan"), device=dev) for _ in range(3))
    ind = torch.full((maxM,), float("nan"), device=dev)
    offs = torch.tensor([off, -1], dtype=torch.int32, device=dev)
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    ops.hypotheses(lg.to(dev), 20, c(kps), c(kpt), c(Rs), c(Rt), c(sm), c(tm), torch.tensor([M], dtype=torch.int32, device=dev), maxM,
                   offs[0:1], offs[1:2], ind, R_acc, t_acc, ss_acc, tt_acc)
    assert int(offs[1].item()) == off + M
    ind = ind.cpu()
    assert torch.isnan(ind[M:]).all()
    for a in (R_acc, t_acc, ss_acc, tt_acc):
        a = a.cpu()
        assert torch.isnan(a[:off]).all() and torch.isnan(a[off + M:]).all() and torch.isfinite(a[off:off + M]).all()
    ind64 = oracle.soft_argmax(torch.from_numpy(logits))
    dind = (ind[:M].double() - ind64).abs()
    assert float(dind.max()) <= 2e-5, float(dind.max())
    assert abs(float(ind[0]) - 9.5) < 1e-6 and abs(float(ind[3]) - 9.5) < 1e-6 and float(ind[1]) < 1e-20 and float(ind[2]) > 19 - 1e-6
    # R and t against the float64 formula at the kernel's own bin (fp32 trigonometry and products only) ...
    s_i, t_i = torch.from_numpy(sm[:M].astype(np.int64)), torch.from_numpy(tm[:M].astype(np.int64))
    args = (torch.from_numpy(kps).double()[s_i], torch.from_numpy(kpt).double()[t_i], torch.from_numpy(Rs).double()[s_i],
            torch.from_numpy(Rt).double()[t_i])
    R64, t64 = oracle.hypotheses(ind[:M].double(), *args)
    Rg, tg = R_acc[off:off + M].cpu().double(), t_acc[off:off + M].cpu().double()
    eR, et = float((Rg - R64).abs().max()), float((tg - t64).abs().max())
    assert eR < 2e-6 and et < 2e-5, (eR, et)
    # ... and at the float64 bin
    R64b, _ = oracle.hypotheses(ind64, *args)
    assert float((Rg - R64b).abs().max()) < 2e-6 + 2 * np.pi / 20 * float(dind.max())
    assert (ss_acc[off:off + M].cpu().numpy() == kps[sm[:M]]).all() and (tt_acc[off:off + M].cpu().numpy() == kpt[tm[:M]]).all()
    report("G5 hypotheses: soft arg-max, R, t", max(float(dind.max()), eR, et))


# ------------------------------------------------------------------------------------------------ G6 bx_concat_matches
@pytest.mark.parametrize("S", [1, 3, 8])
def test_concat_matches_vs_numpy(dev, S):
    """Per-scale lists concatenated in scale order with their row offsets; d_offs holds the prefix sums and the total,
    entries past the total and past d_offs[S] are untouched."""
    from bufferx_b200 import ops
    rng = np.random.default_rng(S)
    stride = 50
    counts = rng.integers(0, stride + 1, S).astype(np.int32)
    counts[0] = stride
    if S > 1:
        counts[1] = 0
    s_lists = rng.integers(0, 1000, (S, stride)).astype(np.int32)
    t_lists = rng.integers(0, 1000, (S, stride)).astype(np.int32)
    s_off = rng.integers(0, 10000, S).astype(np.int32)
    t_off = rng.integers(0, 10000, S).astype(np.int32)
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    s_all = torch.full((S * stride + 4,), -7, dtype=torch.int32, device=dev)
    t_all = torch.full((S * stride + 4,), -7, dtype=torch.int32, device=dev)
    d_offs = torch.full((S + 3,), -7, dtype=torch.int32, device=dev)
    # through the C-ABI with our own output buffers, so that what lies past the total can be checked
    sl, tl, cn = c(s_lists), c(t_lists), c(counts)
    ops._check(ops.load_library().bx_concat_matches(sl.data_ptr(), tl.data_ptr(), cn.data_ptr(), S, stride,
                                                    s_off.ctypes.data_as(ops.c_void_p), t_off.ctypes.data_as(ops.c_void_p),
                                                    s_all.data_ptr(), t_all.data_ptr(), d_offs.data_ptr(), None), "bx_concat_matches")
    torch.cuda.synchronize()
    exp_s = np.concatenate([s_lists[i, :counts[i]] + s_off[i] for i in range(S)])
    exp_t = np.concatenate([t_lists[i, :counts[i]] + t_off[i] for i in range(S)])
    total = int(counts.sum())
    got_s, got_t, got_o = s_all.cpu().numpy(), t_all.cpu().numpy(), d_offs.cpu().numpy()
    assert (got_s[:total] == exp_s).all() and (got_t[:total] == exp_t).all()
    assert (got_s[total:] == -7).all() and (got_t[total:] == -7).all()
    assert (got_o[:S + 1] == np.concatenate([[0], np.cumsum(counts)])).all() and (got_o[S + 1:] == -7).all()
    # the same through the wrapper
    offs = torch.zeros(S + 1, dtype=torch.int32, device=dev)
    ws, wt = ops.concat_matches(c(s_lists), c(t_lists), c(counts), s_off, t_off, offs)
    assert (ws[:total].cpu().numpy() == exp_s).all() and (wt[:total].cpu().numpy() == exp_t).all()
    assert (offs.cpu().numpy() == got_o[:S + 1]).all()


def test_concat_matches_rejects_more_than_eight_scales(dev):
    from bufferx_b200 import ops
    S, K = 9, 4
    z = torch.zeros((S, K), dtype=torch.int32, device=dev)
    with pytest.raises(ops.BufferXError, match="1 <= S <= 8"):
        ops.concat_matches(z, z, torch.zeros(S, dtype=torch.int32, device=dev), [0] * S, [0] * S,
                           torch.zeros(S + 1, dtype=torch.int32, device=dev))
