"""GPU experiment: accuracy of the 3xTF32 tensor-core GEMM against fp64, versus K and accumulation segmenting.
    python tools/tc_precision.py            (needs an H100)"""
import os, sys, ctypes
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bufferx_b200 as bx
from bufferx_b200 import ops

dev = torch.device("cuda:0")
lib = ops.load_library()
g = torch.Generator().manual_seed(0)


def run(K, Cout, n, S, seg, relu_like=True):
    x = torch.randn((n, K, S), generator=g)
    if relu_like:
        x = x.abs()
    W = torch.randn((Cout, K), generator=g) / K ** 0.5
    b = torch.zeros(Cout)
    ref = torch.einsum("ok,nks->nos", W.double(), x.double())
    Wt = W.t().contiguous()[None]                      # [T=1, Cin, Cout]
    lib.bx_conv_tc_set_segment_stages(seg)
    out_cb = torch.empty((n, Cout // 4, S, 4), device=dev)             # the tensor-core kernel takes channel-blocked activations
    ops.conv_layer_tc(ops.GEOM_VALID3D, ops.to_blocked(x.to(dev)), ops.conv_tc_weights(Wt.to(dev)), b.to(dev), out_cb, n, K, Cout,
                      1, 1, S, 1, 1, 1, False)
    out = ops.from_blocked(out_cb)
    err = (out.cpu().double() - ref)
    scale = ref.abs().mean()
    return float(err.abs().max() / scale), float(err.abs().mean() / scale), float(err.mean() / scale), float(ref.mean() / scale)


print("K Cout seg  max/mean|ref|  mean|err|/mean|ref|  mean(err)/mean|ref| (bias)   mean(ref)")
for K in (128, 576, 1152):
    for Cout in (64, 128):
        for seg in (100000, 24, 6, 2):
            for relu_like in (True, False):
                r = run(K, Cout, 64, 140, seg, relu_like)
                print(f"K={K:5d} N={Cout:4d} seg={seg:6d} relu={int(relu_like)}  max={r[0]:.3e} mean={r[1]:.3e} bias={r[2]:+.3e} ref={r[3]:+.2f}")
