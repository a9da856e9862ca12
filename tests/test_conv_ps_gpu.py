"""The per-sample descriptor-stack convolution (csrc/bx_conv_ps.cu, ops.conv_layer_ps) against conv_sd_kernel
(ops.conv_layer_sd) on the same input: every output byte -- values, wrap columns, zero rows, and the rows neither kernel
writes -- must be identical.  Covers every Cylindrical_Net layer shape at the production batch, sample counts at the edges of
the unit schedule, a device sample count below the capacity and the fp16-range flag."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# Cylindrical_Net (models/patchnet.py): (geometry, Cin, Cout, relu, presplit output)
LAYERS = [("3d", 16, 64, True, True), ("2d", 64, 64, True, True), ("2d", 64, 128, True, True), ("2d", 128, 128, True, True),
          ("2d", 128, 64, True, True), ("2d", 64, 64, True, True), ("2d", 64, 32, True, True), ("2d", 32, 32, False, False)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    import bufferx_b200 as bx
    bx.ops.load_library()
    return torch.device("cuda:0")


def _case(dev, n, geom, Cin, Cout, seed, scale=1.0):
    """presplit input image of n samples, the conv_sd weight image and a bias (Cin = 16 with 3d: three radial slices)."""
    from bufferx_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    C = 3 * Cin if geom == "3d" else Cin
    T = 27 if geom == "3d" else 9
    x = torch.relu(torch.randn((n, C, 7, 20), generator=g, device=dev))
    Wt = torch.randn((T, Cin, Cout), generator=g, device=dev) * (scale / (Cin * T) ** 0.5)
    b = torch.randn(Cout, generator=g, device=dev) * 0.1
    return ops.sd_pack(x), ops.conv_sd_weights(Wt), b


def _out(dev, n, Cout, presplit):
    """NaN-filled output of either format, so that bytes a kernel leaves untouched compare too."""
    from bufferx_b200 import ops
    if presplit:
        return torch.full(ops.conv_sd_buffer(n, Cout, dev).shape, float("nan"), dtype=torch.float16, device=dev)
    return torch.full((n, Cout // 4, 140, 4), float("nan"), dtype=torch.float32, device=dev)


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t.view(torch.int32)


def _both(dev, n, layer, seed, d_n=None, scale=1.0, flag=False):
    from bufferx_b200 import ops
    geom, Cin, Cout, relu, presplit = layer
    G = ops.GEOM_CYL3D if geom == "3d" else ops.GEOM_CYL2D
    x, w, b = _case(dev, n, geom, Cin, Cout, seed, scale)
    res = []
    for conv in (ops.conv_layer_sd, ops.conv_layer_ps):
        o = _out(dev, n, Cout, presplit)
        f = torch.zeros(1, dtype=torch.int32, device=dev) if flag else None
        conv(G, x, w, b, o, n, Cin, Cout, relu, f, d_n=d_n)
        torch.cuda.synchronize()
        res.append((o, f))
    return res


@pytest.mark.parametrize("layer", LAYERS, ids=[f"{g}-{ci}-{co}" for g, ci, co, _, _ in LAYERS])
def test_conv_ps_bit_identical_production_batch(dev, layer):
    (ref, _), (got, _) = _both(dev, 9000, layer, seed=1)
    assert torch.equal(_bits(got), _bits(ref)), f"{layer}: {(_bits(got) != _bits(ref)).sum().item()} differing elements"


@pytest.mark.parametrize("n", [1, 2, 7, 131, 263])
@pytest.mark.parametrize("li", [0, 2, 3, 6, 7])
def test_conv_ps_bit_identical_edge_counts(dev, n, li):
    """1, 2, odd, and one less than a multiple of 132 (the H100's SM count = the grid of a large launch) samples."""
    (ref, _), (got, _) = _both(dev, n, LAYERS[li], seed=10 + n)
    assert torch.equal(_bits(got), _bits(ref))


@pytest.mark.parametrize("li", [1, 3, 6, 7])
def test_conv_ps_device_count_below_capacity(dev, li):
    """d_n = 217 of n = 300: both kernels compute and write the first 217 samples (and the zero row after them) only."""
    d_n = torch.tensor([217], dtype=torch.int32, device=dev)
    (ref, _), (got, _) = _both(dev, 300, LAYERS[li], seed=5, d_n=d_n)
    assert torch.equal(_bits(got), _bits(ref))


@pytest.mark.parametrize("li", [1, 3, 6])
def test_conv_ps_fp16_range_flag(dev, li):
    """Activations past fp16 range raise the flag in both kernels (the caller then re-runs the stack on the TF32 kernel);
    in range, neither raises it."""
    (_, f_ref), (_, f_got) = _both(dev, 64, LAYERS[li], seed=7, flag=True)
    assert f_ref.item() == 0 and f_got.item() == 0
    (_, f_ref), (_, f_got) = _both(dev, 64, LAYERS[li], seed=7, scale=4.0e5, flag=True)
    assert f_ref.item() == 1 and f_got.item() == 1


def test_conv_ps_refuses_fp32_input(dev):
    """The per-sample kernel has no fp32 loader: an fp32 input is an error, not a silent fall-back."""
    from bufferx_b200 import ops
    x = torch.zeros((2, 16, 140, 4), device=dev)
    with pytest.raises(ops.BufferXError):
        ops.conv_layer_ps(ops.GEOM_CYL2D, x, torch.zeros(9 * 64 * 64, dtype=torch.float16, device=dev), torch.zeros(64, device=dev),
                          _out(dev, 2, 64, True), 2, 64, 64, True)


def test_cylindrical_net_runs_the_per_sample_kernel(dev, monkeypatch):
    """Cylindrical_Net.forward on a presplit input calls conv_layer_ps for every layer but the fp32-output last one, and its
    result equals the same stack run layer by layer on conv_sd_kernel (ops.conv_layer_sd) bit for bit."""
    import bufferx_b200 as bx
    from bufferx_b200 import ops
    from bufferx_b200.synth import init_synthetic_weights, workload_cfg
    net = init_synthetic_weights(bx.BufferX(workload_cfg("C2"))).cuda().Desc.conv_net
    K = 517
    x = ops.sd_pack(torch.relu(torch.randn((K, 48, 7, 20), device=dev)))
    calls = []
    real = ops.conv_layer_ps
    monkeypatch.setattr(ops, "conv_layer_ps", lambda *a, **k: (calls.append(1), real(*a, **k))[1])
    got, _ = net(x, K=K)
    assert len(calls) == len(net.layers) - 1
    L = net.folded()
    ref = x
    for i, l in enumerate(L):
        out = ops.conv_sd_buffer(K, l["cout"], dev) if i < len(L) - 1 else torch.empty((K, l["cout"] // 4, 140, 4), device=dev)
        ref = ops.conv_layer_sd(ops.GEOM_CYL3D if i == 0 else ops.GEOM_CYL2D, ref, l["w_sd"], l["b"], out, K, l["cin"], l["cout"],
                                l["relu"])
    assert torch.equal(_bits(got), _bits(ref))
