"""The channels-as-M form of the shifted-descriptor convolution (csrc/bx_conv_sd.cu, presplit input with Cout <= 64): each MMA
warpgroup owns a whole 128-row tile, a CTA works on two tiles, and Cout <= 32 runs through the P / Q weight images.  Each case
is checked against torch fp32 at the bound of the other conv_sd tests."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def _wt(W, dev):
    from bufferx_b200 import ops
    return ops.conv_sd_weights(W.reshape(W.shape[0], W.shape[1], -1).permute(2, 1, 0).contiguous().to(dev))


def _rel(a, b):
    return float((a.cpu() - b).abs().max() / b.abs().max())


def _cyl_case(seed, n, Cin, Cout):
    from oracle import oracle as O
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((n, Cin, 7, 20), generator=g)
    W = torch.randn((Cout, Cin, 3, 3), generator=g) / (Cin * 9) ** 0.5
    b = torch.randn(Cout, generator=g) * 0.1
    return x, W, b, F.relu(F.conv2d(O._pad_cyl(x), W, b))


@pytest.mark.parametrize("n,Cin,Cout", [(3, 64, 64), (5, 32, 32), (1, 16, 64), (9, 64, 20)])
def test_conv_sd_odd_tile_count(dev, n, Cin, Cout):
    """n * 176 rows = an odd number of 128-row tiles (n = 1: two tiles): the last unit's second warpgroup has no tile of its own.
    The rows of every sample are right."""
    from bufferx_b200 import ops
    assert ((n * 176 + 127) // 128) % 2 == (0 if n == 1 else 1)
    x, W, b, y = _cyl_case(100 + n, n, Cin, Cout)
    xs, w, bd = ops.sd_pack(x.to(dev)), _wt(W, dev), b.to(dev)
    o = torch.full((n, Cout // 4, 140, 4), float("nan"), device=dev)
    ops.conv_layer_sd(ops.GEOM_CYL2D, xs, w, bd, o, n, Cin, Cout, True)
    assert _rel(ops.from_blocked(o).view(n, Cout, 7, 20), y) < 2e-5


def test_conv_sd_cin128_cout64_streamed_weights(dev):
    """128 -> 64: the 288 KB weight image does not fit next to the activation ring and streams through a ring of three-tap
    stages, each released only when both warpgroups have used it.  Presplit out, then back to fp32 through a 64 -> 64 layer."""
    from bufferx_b200 import ops
    from oracle import oracle as O
    n = 41
    x, W, b, y = _cyl_case(7, n, 128, 64)
    img = ops.conv_sd_buffer(n, 64, dev)
    img.fill_(float("nan"))
    ops.conv_layer_sd(ops.GEOM_CYL2D, ops.sd_pack(x.to(dev)), _wt(W, dev), b.to(dev), img, n, 128, 64, True)
    val, xp = ops.sd_unpack(img, n)
    assert _rel(val, y) < 2e-5
    assert (xp[:, :, 0] == 0).all() and (xp[:, :, 1:, 0] == xp[:, :, 1:, 20]).all() and (xp[:, :, 1:, 21] == xp[:, :, 1:, 1]).all()
    g = torch.Generator().manual_seed(8)
    W2 = torch.randn((64, 64, 3, 3), generator=g) / (64 * 9) ** 0.5
    b2 = torch.randn(64, generator=g) * 0.1
    y2 = F.conv2d(O._pad_cyl(y), W2, b2)
    o = torch.full((n, 16, 140, 4), float("nan"), device=dev)
    ops.conv_layer_sd(ops.GEOM_CYL2D, img, _wt(W2, dev), b2.to(dev), o, n, 64, 64, False)
    assert _rel(ops.from_blocked(o).view(n, 64, 7, 20), y2) < 3e-5


@pytest.mark.parametrize("Cout", [20, 32])
def test_conv_sd_pq_weight_images(dev, Cout):
    """Cout <= 32: the P / Q image is the A operand of the presplit-input kernel and, read with a 256-byte core-matrix stride,
    the B operand of the fp32-input kernel; both give the layer."""
    from bufferx_b200 import ops
    n, Cin = 37, 64
    x, W, b, y = _cyl_case(Cout, n, Cin, Cout)
    w = _wt(W, dev)
    assert w.numel() == Cin // 16 * 9 * 2 * 2 * 64 * 8
    for xin in (ops.sd_pack(x.to(dev)), ops.to_blocked(x.to(dev).reshape(n, Cin, 140))):
        o = torch.full((n, Cout // 4, 140, 4), float("nan"), device=dev)
        ops.conv_layer_sd(ops.GEOM_CYL2D, xin, w, b.to(dev), o, n, Cin, Cout, True)
        assert _rel(ops.from_blocked(o).view(n, Cout, 7, 20), y) < 2e-5, xin.dtype
    if Cout % 16 == 0:       # presplit out of the Cout 32 form
        img = ops.conv_sd_buffer(n, Cout, dev)
        img.fill_(float("nan"))
        ops.conv_layer_sd(ops.GEOM_CYL2D, ops.sd_pack(x.to(dev)), w, b.to(dev), img, n, Cin, Cout, True)
        val, xp = ops.sd_unpack(img, n)
        assert _rel(val, y) < 2e-5 and (xp[:, :, 0] == 0).all()


def test_conv_sd_valid_raster_cout32_chain(dev):
    """CostNet's 64 -> 32 and 32 -> 32 k = (3,1,3) layers on un-padded rasters with a device-side sample count below the
    capacity: presplit between the layers, samples beyond the count untouched."""
    from bufferx_b200 import ops
    g = torch.Generator().manual_seed(11)
    n, cap = 29, 40
    x = torch.randn((n, 64, 14, 1, 14), generator=g)
    W1 = torch.randn((32, 64, 3, 1, 3), generator=g) / (64 * 9) ** 0.5
    W2 = torch.randn((32, 32, 3, 1, 3), generator=g) / (32 * 9) ** 0.5
    b1, b2 = torch.randn(32, generator=g) * 0.1, torch.randn(32, generator=g) * 0.1
    y1 = F.relu(F.conv3d(x, W1, b1))
    y2 = F.relu(F.conv3d(y1, W2, b2))
    d_n = torch.tensor([n], dtype=torch.int32, device=dev)
    xin = ops.conv_sd_buffer(cap, 64, dev, 14 * 14).zero_()
    # presplit input over the 14 x 14 raster: [chunk][split][kcore][row][8], row = sample * 196 + position
    flat = torch.zeros((xin.shape[2], 64), device=dev)
    flat[: n * 196] = x.to(dev).reshape(n, 64, 196).permute(0, 2, 1).reshape(n * 196, 64)
    hi = flat.half()
    lo = ((flat - hi.float()) * 2048.0).half()
    xin.copy_(torch.stack([hi, lo], 0).view(2, -1, 4, 2, 8).permute(2, 0, 3, 1, 4).reshape(xin.shape))
    mid = ops.conv_sd_buffer(cap, 32, dev, 12 * 12)
    mid.fill_(float("nan"))
    ops.conv_layer_sd(ops.GEOM_VALID3D, xin, _wt(W1, dev), b1.to(dev), mid, cap, 64, 32, True, None, d_n=d_n, D=14, W=14)
    out = torch.full((cap, 8, 100, 4), float("nan"), device=dev)
    ops.conv_layer_sd(ops.GEOM_VALID3D, mid, _wt(W2, dev), b2.to(dev), out, cap, 32, 32, True, None, d_n=d_n, D=12, W=12)
    got = ops.from_blocked(out[:n]).view(n, 32, 10, 1, 10).cpu()
    assert float((got - y2).abs().max() / y2.abs().max()) < 3e-5
    assert torch.isnan(out[n:]).all()
