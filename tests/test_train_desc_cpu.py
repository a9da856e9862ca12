"""CPU checks of the Desc training step: what ptxas makes of csrc/bx_train_desc.cu (the cylindrical convolution kernels run on
DMMA, no kernel spills or keeps a stack frame), and the float64 oracle (oracle/train_desc.py) against torch's own modules in
training mode: outputs, running statistics and gradients."""
import importlib.util
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "buffer-x_b200", "csrc")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    spec = importlib.util.spec_from_file_location("_bx_build_flags", os.path.join(CSRC, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    nvcc = b._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)) and shutil.which(nvcc) is None:
        pytest.skip("nvcc not available")
    obj = str(tmp_path_factory.mktemp("train_desc") / "bx_train_desc.o")
    r = subprocess.run([nvcc] + b.ARCH + b.COMMON + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "bx_train_desc.cu"), "-o", obj],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.isabs(nvcc) else shutil.which("cuobjdump")
    return cuobjdump, obj, r.stdout + r.stderr


def test_no_kernel_spills_or_keeps_a_stack_frame(compiled):
    _, _, log = compiled
    frames = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert len(frames) >= 12, log
    bad = [f for f in frames if any(int(v) for v in f[1:])]
    assert not bad, bad


def test_cylindrical_convolutions_run_on_dmma(compiled):
    cuobjdump, obj, _ = compiled
    if not cuobjdump or not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    conv = [f for f in funcs if "cyl_mma_kernel" in f.split("\n", 1)[0] or "cyl_wgrad_kernel" in f.split("\n", 1)[0]]
    assert len(conv) == 3, [f.split("\n", 1)[0] for f in funcs]
    for f in conv:
        assert "DMMA.16x8x16" in f, f.split("\n", 1)[0]


class _Desc(nn.Module):
    """MiniSpinNet's trainable layers in torch's own modules (patch_embedder.py:16-42, patchnet.py:68-84)."""

    def __init__(self):
        super().__init__()
        self.pnt_layer = nn.Sequential(nn.Conv2d(3, 16, 1), nn.BatchNorm2d(16), nn.ReLU(True))
        self.pool_layer = nn.Sequential(nn.Conv2d(32, 16, 1), nn.BatchNorm2d(16), nn.ReLU(True), nn.Conv2d(16, 1, 1), nn.BatchNorm2d(1),
                                        nn.ReLU(True))
        spec = [(16, 64, 3), (64, 64, 2), (64, 128, 2), (128, 128, 2), (128, 64, 2), (64, 64, 2), (64, 32, 2), (32, 32, 2)]
        ops = []
        for i, (ci, co, d) in enumerate(spec):
            ops.append(nn.Conv3d(ci, co, 3) if d == 3 else nn.Conv2d(ci, co, 3))
            if i < 7:
                ops += [nn.BatchNorm3d(co, affine=False) if d == 3 else nn.BatchNorm2d(co, affine=False), nn.ReLU(True)]
        self.conv_net = nn.Module()
        self.conv_net.ops = nn.ModuleList(ops)

    def forward(self, inv):
        from oracle import oracle as O
        x = inv.permute(0, 3, 1, 2)
        x = F.max_pool2d(self.pnt_layer(x), kernel_size=(1, x.shape[3])).squeeze(3)
        K = x.shape[0]
        x = x.view(K, 16, 3, 7, 20)
        for i, m in enumerate(self.conv_net.ops):
            x = m(O._pad_cyl(x)) if isinstance(m, (nn.Conv2d, nn.Conv3d)) else m(x)
            if i == 2:                                             # after the first layer's ReLU: the depth is collapsed
                x = x.squeeze(2)
        w = self.pool_layer(x)
        f = F.avg_pool2d(x * w, kernel_size=(7, 20)).view(K, -1)
        return F.normalize(f, dim=1), F.normalize(x, dim=1)


def test_oracle_matches_torch_modules_in_training_mode():
    from oracle import train_desc as TD
    from oracle.train_step import bn_hparams, state64
    torch.manual_seed(0)
    net = _Desc().double().train()
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, nn.BatchNorm2d) and m.affine:
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
    sd = {"Desc." + k: v.detach().clone() for k, v in net.state_dict().items()}
    rng = np.random.default_rng(1)
    invs = [rng.standard_normal((6, 420, 10, 3)).astype(np.float32) * 0.3 for _ in range(2)]
    for inv in invs:
        inv[:, :, 8:] = 0.0                                        # zero slots
        inv[:, :, 1] = inv[:, :, 0]                                # a duplicated sample
    inv[0] = 0.0                                                   # an all-zero patch
    hp = {"Desc." + k: v for k, v in bn_hparams(net).items()}
    params, st, stats = TD.desc_params(sd), state64(sd), []
    outs = [TD.desc_train(v, params, st, stats, hp) for v in invs]
    refs = [net(torch.from_numpy(v).double()) for v in invs]
    kpt = rng.standard_normal((6, 3)) * 0.05
    label = rng.integers(0, 20, 6)
    loss = TD.desc_loss(outs[0][0], outs[1][0], kpt, TD.equi_match(outs[0][1], outs[1][1]), label)
    ref_loss = TD.desc_loss(refs[0][0], refs[1][0], kpt, TD.equi_match(refs[0][1], refs[1][1]), label)
    assert torch.allclose(loss, ref_loss, rtol=1e-12, atol=0)
    loss.backward()
    ref_loss.backward()
    named = dict(net.named_parameters())
    assert set(params) == set(named)
    scale = max(float(p.grad.abs().max()) for p in named.values())   # the biases before a BatchNorm: analytically zero
    for k, p in params.items():
        assert torch.allclose(p.grad, named[k].grad, rtol=1e-9, atol=1e-12 * scale), k
    msd = net.state_dict()
    for k, v in msd.items():
        o = st["Desc." + k]
        assert torch.equal(o, v) if not v.is_floating_point() else torch.allclose(o, v, rtol=1e-12, atol=1e-15), k
