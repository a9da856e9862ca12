"""CPU checks of the channels-as-M form of the shifted-descriptor convolution (csrc/bx_conv_sd.cu): the presplit-input kernels
with Cout <= 64 issue only m64n128k16 wgmmas (output channels as M, a whole 128-row tile as N), and ops.conv_sd_weights lays out
the Cout <= 32 weights as the P / Q images that form relies on."""
import importlib.util
import os
import re
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "buffer-x_b200", "csrc")


def _build_module():
    spec = importlib.util.spec_from_file_location("_bx_build_flags_cm", os.path.join(CSRC, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_presplit_cout64_and_below_issue_m64n128k16_only(tmp_path):
    b = _build_module()
    nvcc = b._nvcc()
    if not (os.path.isabs(nvcc) and os.path.exists(nvcc)) and shutil.which(nvcc) is None:
        pytest.skip("nvcc not available")
    cand = os.path.join(os.path.dirname(nvcc), "cuobjdump") if os.path.isabs(nvcc) else None
    cuobjdump = cand if cand and os.path.exists(cand) else shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump not available")
    obj = str(tmp_path / "bx_conv_sd.o")
    r = subprocess.run([nvcc] + b.ARCH + b.COMMON + ["-c", os.path.join(CSRC, "bx_conv_sd.cu"), "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    r = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    shapes, key = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function : \S*conv_sd_kernelILi(\d+)ELi(\d)ELi(\d)E", line)
        if m:
            key = tuple(int(v) for v in m.groups())                    # (NT, IN_SD, OUT_SD)
            shapes[key] = []
        elif "Function :" in line:
            key = None
        elif key:
            m = re.search(r"HGMMA\.(\d+x\d+x\d+)", line)
            if m:
                shapes[key].append(m.group(1))
    for nt in (32, 64):
        for out_sd in (0, 1):
            got = shapes.get((nt, 1, out_sd))
            assert got, f"no HGMMA found for conv_sd_kernel<{nt}, 1, {out_sd}>"
            assert set(got) == {"64x128x16"}, f"conv_sd_kernel<{nt}, 1, {out_sd}>: {sorted(set(got))}"


@pytest.mark.parametrize("Cin,Cout", [(64, 20), (32, 32)])
def test_cout32_weight_image_is_p_and_q(Cin, Cout):
    """[chunk][tap][kcore][P | Q][64][8]: in each 16-row group w, P = hi / lo and Q = zero / hi of channels 8w..8w+7."""
    import bufferx_b200.ops as ops
    g = torch.Generator().manual_seed(Cout)
    Wt = torch.randn((9, Cin, Cout), generator=g)
    img = ops.conv_sd_weights(Wt).view(Cin // 16, 9, 2, 2, 4, 2, 8, 8).float()   # [chunk, tap, kcore, P|Q, w, split, 8 ch, 8 k]
    P, Q = img[:, :, :, 0], img[:, :, :, 1]
    # back to [tap, Cin, 32]: k = chunk * 16 + kcore * 8 + kk, n = 8 w + channel
    back = lambda t: t.permute(1, 0, 2, 5, 3, 4).reshape(9, Cin, 32)
    W = torch.zeros((9, Cin, 32))
    W[:, :, :Cout] = Wt
    hi, lo = back(P[:, :, :, :, 0]), back(P[:, :, :, :, 1])
    assert torch.equal(hi, W.half().float())
    assert torch.equal(lo, ((W - W.half().float()) * 2048.0).half().float())
    assert (Q[:, :, :, :, 0] == 0).all() and torch.equal(back(Q[:, :, :, :, 1]), hi)
