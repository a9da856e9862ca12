"""Parameter containers + weight folding for the two convolution stacks.

Mirrors the state_dict layout of /root/reference/models/patchnet.py: ``Cylindrical_Net``
(:68-84, ops.{0,1,3,4,...,21}) and ``CostNet`` (:192-210, ops.{0,1,...,27}); BatchNorm layers in the
stacks have ``affine=False`` (:28,31).  The modules hold parameters only -- the arithmetic runs in
the library's convolution kernels (``bx_conv_layer_sd``, ``bx_conv_layer_tc``, ``bx_costvol_ab``).  ``folded()``
returns, per conv layer, the weight re-laid as [tap][Cin][Cout] with the eval-mode BatchNorm folded in (computed in
fp64, stored fp32), and the kernels' operand images of it.
"""
import torch
import torch.nn as nn

import os

from bufferx_b200 import ops

# BX_CONV=tc: the descriptor stack on the TF32 kernel (bx_conv_tc.cu) instead of the shifted-descriptor fp16-split
# kernel (bx_conv_sd.cu, the default).  The TF32 kernel is also the automatic fall-back when an activation leaves fp16 range.
USE_TF32_DESC = os.environ.get("BX_CONV", "sd").lower() == "tc"
# BX_SD_DYNAMIC=1: the persistent conv kernels draw their tiles from a device-side counter (bx_conv_layer_sd d_tile_ctr) instead
# of the static stride.  It brought no gain with six pairs in flight (a launch whose CTAs start late still cannot finish before
# they have been scheduled), so the static stride stays the default; that was measured on the B200 and has not been
# re-measured on the H100.  The path is kept and tested.
DYNAMIC_TILES = os.environ.get("BX_SD_DYNAMIC", "0") == "1"


def fold_conv_bn(conv_w, conv_b, bn_mean=None, bn_var=None, bn_w=None, bn_b=None, eps=1e-5):
    """-> (Wt [T, Cin, Cout] f32 contiguous, bias [Cout] f32).  Works for 1x1/2-D/3-D kernels."""
    W = conv_w.detach().double()
    b = conv_b.detach().double()
    Cout, Cin = W.shape[0], W.shape[1]
    W = W.reshape(Cout, Cin, -1)
    if bn_mean is not None:
        s = 1.0 / torch.sqrt(bn_var.detach().double() + eps)
        if bn_w is not None:
            s = s * bn_w.detach().double()
        W = W * s[:, None, None]
        b = (b - bn_mean.detach().double()) * s
        if bn_b is not None:
            b = b + bn_b.detach().double()
    Wt = W.permute(2, 1, 0).contiguous().float()
    return Wt, b.float().contiguous()


class _ConvStack(nn.Module):
    """ModuleList ``ops`` with the reference's index layout: conv, [bn], [relu], conv, ..."""

    def __init__(self, spec, bn_affine=False):
        super().__init__()
        self.ops = nn.ModuleList([])
        self.layers = []  # (conv index, bn index or None, relu?)
        for (cin, cout, k, bn, relu) in spec:
            ci = len(self.ops)
            if len(k) == 3:
                self.ops.append(nn.Conv3d(cin, cout, kernel_size=tuple(k)))
            else:
                self.ops.append(nn.Conv2d(cin, cout, kernel_size=tuple(k)))
            bi = None
            if bn:
                bi = len(self.ops)
                self.ops.append((nn.BatchNorm3d if len(k) == 3 else nn.BatchNorm2d)(cout, affine=bn_affine))
            if relu:
                self.ops.append(nn.ReLU(inplace=True))
            self.layers.append((ci, bi, relu))
        self._folded = None
        self.sd_kernel_sizes = ()    # kernel sizes whose layers also get the fp16-split weight image of bx_conv_layer_sd

    def invalidate(self):
        self._folded = None

    def _apply(self, fn, *a, **k):
        self._folded = None
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self._folded = None
        return super()._load_from_state_dict(*a, **k)

    def folded(self):
        if self._folded is None:
            out = []
            for (ci, bi, relu) in self.layers:
                conv = self.ops[ci]
                bn = self.ops[bi] if bi is not None else None
                Wt, b = fold_conv_bn(conv.weight, conv.bias,
                                     None if bn is None else bn.running_mean, None if bn is None else bn.running_var,
                                     None if bn is None or not bn.affine else bn.weight,
                                     None if bn is None or not bn.affine else bn.bias,
                                     eps=1e-5 if bn is None else bn.eps)
                ks = tuple(conv.kernel_size)
                kk = ks if len(ks) == 3 else (1,) + ks
                sd_ok = Wt.is_cuda and kk in self.sd_kernel_sizes and conv.in_channels % 16 == 0 and conv.out_channels % 16 == 0
                out.append(dict(w=Wt, w_tc=ops.conv_tc_weights(Wt) if Wt.is_cuda else None, w_sd=ops.conv_sd_weights(Wt) if sd_ok else None,
                                b=b, cin=conv.in_channels, cout=conv.out_channels, k=kk, relu=relu))
            self._folded = out
        return self._folded


class Cylindrical_Net(_ConvStack):
    """[K,16,3,7,20] -> [K,32,7,20]  (reference: models/patchnet.py:68-84)."""

    def __init__(self, inchan=16, dim=32):
        spec = [(inchan, 64, (3, 3, 3), True, True), (64, 64, (3, 3), True, True), (64, 128, (3, 3), True, True),
                (128, 128, (3, 3), True, True), (128, 64, (3, 3), True, True), (64, 64, (3, 3), True, True),
                (64, 32, (3, 3), True, True), (32, dim, (3, 3), False, False)]
        super().__init__(spec)
        self.out_dim = dim
        self.sd_kernel_sizes = ((1, 3, 3), (3, 3, 3))
        self.force_tf32 = USE_TF32_DESC      # set (sticky) by BufferX when the fp16-range flag fired once
        self._flag = None

    def overflow_flag(self, dev):
        """int32[1] on `dev`, OR-ed by bx_conv_layer_sd when an activation is outside fp16 range (sticky until cleared)."""
        if self._flag is None or self._flag.device != dev:
            self._flag = torch.zeros(1, dtype=torch.int32, device=dev)
        return self._flag

    def forward(self, x, K=None, d_n=None):
        """x [K,4,420,4] channel-blocked (or the presplit image of K patches) -> (x_out [K,8,140,4], None).
        d_n: optional int32[1] CUDA count: only the first min(d_n, K) samples are computed (the rest of x_out is undefined)."""
        presplit_in = x.dtype == torch.float16             # [3, 4, rows, 8] from bx_spt_pnt_sd: K is passed separately
        K = x.shape[0] if not presplit_in else int(K)
        dev = x.device
        L = self.folded()
        cur = x.contiguous()
        use_sd = not self.force_tf32
        assert use_sd or not presplit_in
        flag = self.overflow_flag(dev) if use_sd else None
        # dynamic tile scheduling of the persistent conv kernels: one zeroed counter pair per layer (and per call = per stream)
        ctrs = torch.zeros(2 * len(L), dtype=torch.int32, device=dev) if (use_sd and DYNAMIC_TILES) else None
        for i, l in enumerate(L):
            out = torch.empty((K, l["cout"] // 4, 140, 4), dtype=torch.float32, device=dev)
            if use_sd:       # layer-to-layer activations in the presplit padded fp16 format; fp32 in at the first, fp32 out at the last layer
                out = out if i == len(L) - 1 else ops.conv_sd_buffer(K, l["cout"], dev)
                ops.conv_layer_sd(ops.GEOM_CYL3D if i == 0 else ops.GEOM_CYL2D, cur, l["w_sd"], l["b"], out, K, l["cin"], l["cout"], l["relu"], flag,
                                  d_n=d_n, tile_ctr=None if ctrs is None else ctrs[2 * i:2 * i + 2])
                cur = out
                continue
            if i == 0:
                ops.conv_layer_tc(ops.GEOM_CYL3D, cur, l["w_tc"], l["b"], out, K, l["cin"], l["cout"], 3, 7, 20, 3, 3, 3, l["relu"], d_n=d_n)
            else:
                ops.conv_layer_tc(ops.GEOM_CYL2D, cur, l["w_tc"], l["b"], out, K, l["cin"], l["cout"], 1, 7, 20, 1, 3, 3, l["relu"], d_n=d_n)
            cur = out
        return cur, None


class CostNet(_ConvStack):
    """[M,32,20,5,20] cost volume -> [M,20] logits (reference: models/patchnet.py:192-210)."""

    def __init__(self, inchan=32, dim=1):
        spec = [(inchan, 32, (3, 3, 3), True, True), (32, 64, (3, 3, 3), True, True), (64, 64, (3, 1, 3), True, True),
                (64, 128, (3, 1, 3), True, True), (128, 128, (3, 1, 3), True, True), (128, 64, (3, 1, 3), True, True),
                (64, 64, (3, 1, 3), True, True), (64, 32, (3, 1, 3), True, True), (32, 32, (3, 1, 3), True, True),
                (32, dim, (2, 1, 2), False, False)]
        super().__init__(spec)
        self.out_dim = dim
        self.sd_kernel_sizes = ((3, 1, 3),)
        self.force_tf32 = USE_TF32_DESC
        self.flag_source = None          # set by BufferX: the descriptor stack's overflow_flag (one sticky flag per model)

    def forward_matches(self, equi_s, equi_t, s_mids, t_mids, d_M, maxM):
        """equi_* [K,32,7,20]; match lists + device count -> logits [maxM, dim] (rows >= *d_M undefined).
        The k = (3,1,3) layers with Cout >= 32 run on the shifted-descriptor fp16-split kernel (bx_conv_layer_sd, valid
        rasters, presplit activations between them); the factorised first layers and the 2x1x2 head on bx_conv_layer_tc."""
        dev = equi_s.device
        L = self.folded()
        D, H, W = 20, 5, 20
        cur = None
        use_sd = not self.force_tf32
        flag = self.flag_source(dev) if (use_sd and self.flag_source is not None) else None
        ctrs = torch.zeros(2 * len(L), dtype=torch.int32, device=dev) if (use_sd and DYNAMIC_TILES) else None
        for i, l in enumerate(L):
            kd, kh, kw = l["k"]
            OD, OH, OW = D - kd + 1, H - kh + 1, W - kw + 1
            if use_sd and l.get("w_sd") is not None and H == 1 and cur is not None:
                nxt = L[i + 1] if i + 1 < len(L) else None
                nxt_sd = nxt is not None and nxt.get("w_sd") is not None
                out = (ops.conv_sd_buffer(maxM, l["cout"], dev, OD * OW) if nxt_sd
                       else torch.empty((maxM, l["cout"] // 4, OD * OW, 4), dtype=torch.float32, device=dev))
                ops.conv_layer_sd(ops.GEOM_VALID3D, cur, l["w_sd"], l["b"], out, maxM, l["cin"], l["cout"], l["relu"], flag, d_n=d_M, D=D, W=W,
                                  tile_ctr=None if ctrs is None else ctrs[2 * i:2 * i + 2])
                cur, D, H, W = out, OD, OH, OW
                continue
            if i == 0:
                # first layer is linear in the cost volume before its ReLU: two small convolutions of the equivariant
                # maps (bx_costvol_ab); the second layer's loader rebuilds relu(A - B) on the fly (GEOM_COSTAB)
                if "wa" not in l:
                    l["wa"], l["wb"] = ops.costvol_factor_weights(l["w"])
                fa, fb = ops.costvol_ab(equi_s, equi_t, s_mids, t_mids, d_M, maxM, l["wa"], l["wb"], l["b"])
                D, H, W = OD, OH, OW
                continue
            # tensor-core layers exchange channel-blocked activations [maxM, C/4, positions, 4]
            def _f32_out():
                return torch.empty((maxM, l["cout"] // 4, OD * OH * OW, 4), dtype=torch.float32, device=dev)
            if i == 1 and use_sd:       # regenerated first activation -> 96 -> 64 conv over the 18 x 18 raster
                if "w_sd_ab" not in l:
                    l["w_sd_ab"] = ops.conv_sd_weights_costab(l["w"])
                out = ops.conv_sd_buffer(maxM, 64, dev, 256) if L[2].get("w_sd") is not None else _f32_out()
                ops.conv_layer_sd_costab(fa, fb, l["w_sd_ab"], l["b"], out, maxM, l["relu"], flag, d_n=d_M)
                cur, D, H, W = out, OD, OH, OW
                continue
            out = _f32_out()
            if i == 1:
                ops.conv_layer_tc(ops.GEOM_COSTAB, None, l["w_tc"], l["b"], out, maxM, l["cin"], l["cout"], D, H, W, kd, kh, kw, l["relu"],
                                  d_n=d_M, equi_s=fa, equi_t=fb)
            else:
                ops.conv_layer_tc(ops.GEOM_VALID3D, cur, l["w_tc"], l["b"], out, maxM, l["cin"], l["cout"], D, H, W, kd, kh, kw, l["relu"],
                                  d_n=d_M)
            cur, D, H, W = out, OD, OH, OW
        return cur.view(maxM, L[-1]["cout"])      # one output position: blocked [maxM, C/4, 1, 4] == [maxM, C]
