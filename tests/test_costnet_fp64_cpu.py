"""CostNet (a11) against float64 without a GPU: the factorisation of the first layer (bx_costvol_ab), the weight image of the
second layer on the shifted-descriptor kernel (ops.conv_sd_weights_costab) and the float64 oracle functions
(oracle.costnet_fp64, oracle.soft_argmax)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F


@pytest.fixture(scope="module")
def nets():
    """CostNet state_dicts and folded layers: the fitted weights and the seeded random ones."""
    import bufferx_b200 as bx
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    out = {}
    for name, fitted in (("fitted", True), ("random", False)):
        model = init_synthetic_weights(bx.BufferX(workload_cfg("C2")), trained_pose=fitted)
        sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
        out[name] = dict(sd=sd, L=model.Pose.conv.folded())
    return out


def maps(M, seed, shift=3, noise=1e-3):
    """L2-normalised equivariant maps d1, d2 [M,32,5,20] (elevation rows 1..5 of [M,32,7,20]); d2 is d1 rolled by `shift`
    azimuth bins plus noise, renormalised (a true match: the cost volume is ~0 at one n)."""
    g = torch.Generator().manual_seed(seed)
    e1 = F.normalize(torch.randn(M, 32, 7, 20, generator=g), dim=1)
    e2 = F.normalize(torch.roll(e1, shift, dims=3) + noise * torch.randn(M, 32, 7, 20, generator=g), dim=1)
    return e1[:, :, 1:6].contiguous(), e2[:, :, 1:6].contiguous()


def cost_parts(d1, d2, azi_n=20):
    """The two halves of the explicit cost volume [M,C,n,k,l]: d1[c,k,(l-n) mod 20] and d2[c,k,l] (oracle.cost_volume)."""
    M, C, H, _ = d1.shape
    l = torch.arange(azi_n)
    idx = (l[None, :] - l[:, None]) % azi_n
    v1 = d1[:, :, :, idx.reshape(-1)].reshape(M, C, H, azi_n, azi_n).permute(0, 1, 3, 2, 4)
    v2 = d2.unsqueeze(2).expand(M, C, azi_n, H, azi_n)
    return v1, v2


def w5(Wt, k):
    """Folded [T, Cin, Cout] -> conv weight [Cout, Cin, *k]."""
    return Wt.permute(2, 1, 0).reshape(Wt.shape[2], Wt.shape[1], *k)


def factors_fp64(d1, d2, wa, wb, bias):
    """A [M,32,3,20], B [M,32,3,18] of bx_costvol_ab in float64 from the given maps and fp32 factor weights."""
    x1 = d1.double()
    x1 = torch.cat([x1[..., -2:], x1, x1[..., :2]], dim=-1)                 # circular: column j -> azimuth (j - 2) mod 20
    A = F.conv2d(x1, wa.double().permute(3, 0, 1, 2)) + bias.double().view(1, -1, 1, 1)
    B = F.conv2d(d2.double(), wb.double().permute(3, 0, 1, 2))
    return A, B


def regenerate(A, B):
    """relu(A[c,k,(l-n) mod 20] - B[c,k,l]) -> [M,32,18(n),3(k),18(l)]."""
    n = torch.arange(18).view(18, 1)
    l = torch.arange(18).view(1, 18)
    a = A[:, :, :, (l - n) % 20]                                              # [M,32,k,n,l]
    return torch.relu(a - B[:, :, :, None, :]).permute(0, 1, 3, 2, 4)


@pytest.mark.parametrize("net", ["fitted", "random"])
def test_factorised_first_layer_equals_the_direct_convolution(nets, net):
    from bufferx_b200 import ops
    L0 = nets[net]["L"][0]
    wa, wb = ops.costvol_factor_weights(L0["w"])
    for d1, d2 in (maps(24, 1), (4 * torch.randn(24, 32, 5, 20, generator=torch.Generator().manual_seed(2)),
                                 4 * torch.randn(24, 32, 5, 20, generator=torch.Generator().manual_seed(3)))):
        got = regenerate(*factors_fp64(d1, d2, wa, wb, L0["b"]))
        W = w5(L0["w"].double(), (3, 3, 3))
        v1, v2 = cost_parts(d1.double(), d2.double())
        ref = torch.relu(F.conv3d(v1 - v2, W, L0["b"].double()))
        absref = F.conv3d(v1.abs(), W.abs()) + F.conv3d(v2.abs(), W.abs()) + L0["b"].double().abs().view(1, -1, 1, 1, 1)
        ratio = ((got - ref).abs() / absref).max().item()
        assert ratio <= 1e-6, ratio                 # the only rounding is the fp32 storage of wa / wb


def decode_costab(img):
    """ops.conv_sd_weights_costab image [chunk(6)][tap(9)][kcore][split][64][8] -> fp64 [9 taps (dn, dl)][96][64]."""
    v = img.view(6, 9, 2, 2, 64, 8).double()
    w = v[:, :, :, 0] + v[:, :, :, 1] / 2048.0                              # [chunk, tap, kcore, co, 8]
    return w.permute(1, 0, 2, 4, 3).reshape(9, 96, 64)


@pytest.mark.parametrize("net", ["fitted", "random"])
def test_costab_weight_image(nets, net):
    from bufferx_b200 import ops
    L1 = nets[net]["L"][1]
    Wt = L1["w"]                                                              # [27 taps (dn, dk, dl), 32, 64]
    dec = decode_costab(ops.conv_sd_weights_costab(Wt))
    relaid = torch.empty(9, 96, 64, dtype=torch.float64)
    for dn in range(3):
        for dk in range(3):
            for dl in range(3):
                relaid[dn * 3 + dl, dk * 32:(dk + 1) * 32] = Wt[dn * 9 + dk * 3 + dl].double()
    # hi + lo * 2^-11 keeps 22 bits; below fp16's normal range the lo part keeps 2^-35 absolute
    assert ((dec - relaid).abs() <= 2.0 ** -22 * relaid.abs() + 2.0 ** -35).all()

    g = torch.Generator().manual_seed(5)
    x = torch.relu(torch.randn(6, 32, 18, 3, 18, generator=g, dtype=torch.float64))
    ref = F.conv3d(x, w5(Wt.double(), (3, 3, 3)))                          # [M,64,16,1,16]
    xs = x.permute(0, 3, 1, 2, 4).reshape(6, 96, 18, 1, 18)                  # channel dk * 32 + c over the (n, l) raster
    got = F.conv3d(xs, dec.view(3, 1, 3, 96, 64).permute(4, 3, 0, 1, 2))
    absref = F.conv3d(x, w5(Wt.double().abs(), (3, 3, 3)))
    assert ((got - ref).abs() <= 2.0 ** -22 * absref + 1e-12).all()


@pytest.mark.parametrize("net", ["fitted", "random"])
def test_costnet_fp64_and_soft_argmax_against_the_fp32_oracle(nets, oracle, net):
    sd = nets[net]["sd"]
    d1, d2 = maps(40, 7)
    d1b, d2b = maps(40, 9, shift=0)
    d1, d2 = torch.cat([d1, d1b]), torch.cat([d2, d2b])
    M = d1.shape[0]
    ind32 = oracle.cost_volume(d1, d2, sd)
    logits, acts = oracle.costnet_fp64(d1, d2, sd, keep=True)
    assert logits.dtype == torch.float64 and logits.shape == (M, 20)
    assert [tuple(a.shape[1:]) for a in acts] == [(32, 18, 3, 18), (64, 16, 1, 16), (64, 14, 1, 14), (128, 12, 1, 12),
                                                  (128, 10, 1, 10), (64, 8, 1, 8), (64, 6, 1, 6), (32, 4, 1, 4), (32, 2, 1, 2)]
    assert all((a >= 0).all() for a in acts)
    assert torch.equal(oracle.costnet_fp64(d1, d2, sd), logits)
    with torch.no_grad():
        l32, _ = oracle._cost_net(d1, d2, sd, 20, "Pose.conv.")
    lerr = (l32.double() - logits).abs().max(dim=1).values
    assert (lerr <= 2e-5 * logits.abs().max(dim=1).values).all()
    ind64 = oracle.soft_argmax(logits)
    # d ind / d logit_k = p_k (k - ind): a row whose probability mass sits at both ends of the bin range (e.g. bins 0 and
    # 18) turns the same logit error into a larger bin error.  s = sum p_k |k - ind| <= 1 on a single peak.
    p = torch.softmax(logits, dim=1)
    s = (p * (torch.arange(20, dtype=torch.float64)[None] - ind64[:, None]).abs()).sum(dim=1)
    assert ((ind64 - ind32.double()).abs() <= 2e-5 * s.clamp(min=1.0)).all()
    # the expectation is not circular: equal peaks at bins 0 and 19 give 9.5
    two = torch.full((1, 20), -50.0, dtype=torch.float64)
    two[0, 0] = two[0, 19] = 10.0
    assert abs(oracle.soft_argmax(two).item() - 9.5) < 1e-12
    assert abs(oracle.soft_argmax(torch.zeros(1, 20)).item() - 9.5) < 1e-12
