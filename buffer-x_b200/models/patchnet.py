"""Parameter containers + weight folding for the two convolution stacks.

Mirrors the state_dict layout of /root/reference/models/patchnet.py: ``Cylindrical_Net``
(:68-84, ops.{0,1,3,4,...,21}) and ``CostNet`` (:192-210, ops.{0,1,...,27}); BatchNorm layers in the
stacks have ``affine=False`` (:28,31).  The modules hold parameters only -- the arithmetic runs in
the library's convolution kernels (``bx_conv_layer_sd``, ``bx_conv_layer_tc``, ``bx_costvol_ab``).  ``folded()``
returns, per conv layer, the weight re-laid as [tap][Cin][Cout] with the eval-mode BatchNorm folded in (computed in
fp64, stored fp32), and the kernels' operand images of it; the cache is keyed on the versions of the parameters and
buffers, so an optimizer step or a training-mode forward (which moves the running statistics) invalidates it.

Training mode (cfg.stage "Pose", model.train()): ``Cylindrical_Net.forward_train`` runs the convolutions on
``bx_conv_layer_tc`` with the unfolded weights, ``CostNet.forward_train`` on float64 CUDA-core kernels, and both normalise
every BatchNorm'd layer with its batch statistics (bx_train_step.cu), updating the running statistics as torch's BatchNorm
does in training mode.  CostNet's forward sits behind one autograd Function whose backward (bx_ts_conv_backward and the
BatchNorm backward, float64) gives the gradients of every ``ops.*`` weight and bias.
"""
import itertools

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from bufferx_b200 import ops


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


def state_version(module):
    """Identity of the current values of a module's parameters and buffers: changes with every in-place update
    (optimizer.step(), the running statistics of a training-mode forward) and every replacement."""
    return tuple((t.data_ptr(), t._version) for t in itertools.chain(module.parameters(), module.buffers()))


def bn_batch_stats(sums, N, bn, update=True):
    """Per-channel sums [2, C] (sum x, sum x^2, float64) over N samples -> the batch mean and biased variance (float64) that
    a training-mode BatchNorm normalises with; with ``update`` also torch's running update: running_mean <- (1 - m)
    running_mean + m mean, running_var <- (1 - m) running_var + m var N / (N - 1), num_batches_tracked += 1 (m =
    bn.momentum, or the cumulative 1 / num_batches_tracked when it is None)."""
    mean = sums[0] / N
    var = torch.clamp(sums[1] / N - mean * mean, min=0.0)
    if update:
        with torch.no_grad():
            bn.num_batches_tracked += 1
            m = bn.momentum if bn.momentum is not None else 1.0 / float(bn.num_batches_tracked.item())
            bn.running_mean.copy_((1.0 - m) * bn.running_mean.double() + m * mean)
            bn.running_var.copy_((1.0 - m) * bn.running_var.double() + m * var * (N / max(N - 1, 1)))
    return mean, var


def bn_scale_shift(mean, var, bn, dtype=torch.float32):
    """Normalisation by batch statistics as one per-channel affine map (computed in float64, stored as ``dtype``):
    x^ = x scale + shift."""
    scale = 1.0 / torch.sqrt(var + bn.eps)
    if bn.affine:
        scale = scale * bn.weight.detach().double()
    shift = -mean * scale
    if bn.affine:
        shift = shift + bn.bias.detach().double()
    return scale.to(dtype).contiguous(), shift.to(dtype).contiguous()


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
        self._folded_key = None
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
        key = state_version(self)
        if self._folded is None or self._folded_key != key:
            self._folded_key = key
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

    def _layer_train(self, i, x, n, geom, D, H, W):
        """Layer i in training mode on the blocked input x, then (BatchNorm'd layers) the batch statistics and normalise +
        ReLU -> (output, record of what the backward needs).  The descriptor stack (cylindrical geometries) runs the unfolded
        convolution on bx_conv_layer_tc in fp32; CostNet (GEOM_VALID3D) runs in float64 on bx_ts_conv_forward, the
        precision its backward needs."""
        ci, bi, relu = self.layers[i]
        conv = self.ops[ci]
        ks = tuple(conv.kernel_size)
        kd, kh, kw = ks if len(ks) == 3 else (1,) + ks
        f64 = geom == ops.GEOM_VALID3D
        if f64:
            OD, OH, OW = D - kd + 1, H - kh + 1, W - kw + 1
            Wt = conv.weight.detach().double().reshape(conv.out_channels, conv.in_channels, -1).permute(2, 1, 0).contiguous()
            z = ops.conv_forward(x, Wt, conv.bias.detach().double().contiguous(), D, H, W, kd, kh, kw)
        else:
            OD, OH, OW = 1, 7, 20
            Wt, b = fold_conv_bn(conv.weight, conv.bias)
            z = torch.empty((n, conv.out_channels // 4, OD * OH * OW, 4), dtype=torch.float32, device=x.device)
            ops.conv_layer_tc(geom, x, ops.conv_tc_weights(Wt), b, z, n, conv.in_channels, conv.out_channels, D, H, W, kd, kh, kw,
                              relu and bi is None)
        rec = dict(x=x, z=z, Wt=Wt, geom=(D, H, W, kd, kh, kw), out=(OD, OH, OW))
        if bi is None:
            return z, rec
        bn = self.ops[bi]
        N = n * OD * OH * OW
        mean, var = bn_batch_stats(ops.channel_sums(z), N, bn)
        scale, shift = bn_scale_shift(mean, var, bn, z.dtype)
        y = ops.bn_apply(z, scale, shift, relu)
        rec.update(scale=scale, y=y, batch_mean=mean, batch_var=var)
        return y, rec


class Cylindrical_Net(_ConvStack):
    """[K,16,3,7,20] -> [K,32,7,20]  (reference: models/patchnet.py:68-84)."""

    def __init__(self, inchan=16, dim=32):
        spec = [(inchan, 64, (3, 3, 3), True, True), (64, 64, (3, 3), True, True), (64, 128, (3, 3), True, True),
                (128, 128, (3, 3), True, True), (128, 64, (3, 3), True, True), (64, 64, (3, 3), True, True),
                (64, 32, (3, 3), True, True), (32, dim, (3, 3), False, False)]
        super().__init__(spec)
        self.out_dim = dim
        self.sd_kernel_sizes = ((1, 3, 3), (3, 3, 3))
        self.force_tf32 = False      # run on the TF32 kernel (bx_conv_tc.cu); set (sticky) by BufferX when the fp16-range flag fired once
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
        for i, l in enumerate(L):
            out = torch.empty((K, l["cout"] // 4, 140, 4), dtype=torch.float32, device=dev)
            if use_sd:       # layer-to-layer activations in the presplit padded fp16 format; fp32 in at the first, fp32 out at the last layer
                out = out if i == len(L) - 1 else ops.conv_sd_buffer(K, l["cout"], dev)
                # presplit input and output: the per-sample kernel.  conv_sd_kernel keeps an fp32 first-layer input (its loader
                # warps) and the fp32-output last layer, whose two-chunk mainloop is too short to pay for the per-sample epilogue
                # (DESIGN.md section 5: 3.5 % slower on the per-sample kernel)
                conv = ops.conv_layer_ps if cur.dtype == torch.float16 and out.dtype == torch.float16 else ops.conv_layer_sd
                conv(ops.GEOM_CYL3D if i == 0 else ops.GEOM_CYL2D, cur, l["w_sd"], l["b"], out, K, l["cin"], l["cout"], l["relu"], flag,
                     d_n=d_n)
                cur = out
                continue
            if i == 0:
                ops.conv_layer_tc(ops.GEOM_CYL3D, cur, l["w_tc"], l["b"], out, K, l["cin"], l["cout"], 3, 7, 20, 3, 3, 3, l["relu"], d_n=d_n)
            else:
                ops.conv_layer_tc(ops.GEOM_CYL2D, cur, l["w_tc"], l["b"], out, K, l["cin"], l["cout"], 1, 7, 20, 1, 3, 3, l["relu"], d_n=d_n)
            cur = out
        return cur, None

    def forward_train(self, x, stats=None):
        """Training mode: x [K,4,420,4] channel-blocked features -> [K,8,140,4].  Every BatchNorm normalises with the batch
        statistics over K x 140 positions and updates its running statistics once.  ``stats``: optional list that receives
        (batch mean, batch variance) of each BatchNorm, float64."""
        K = x.shape[0]
        cur = x.contiguous()
        for i in range(len(self.layers)):
            cur, rec = self._layer_train(i, cur, K, ops.GEOM_CYL3D if i == 0 else ops.GEOM_CYL2D, 3 if i == 0 else 1, 7, 20)
            if stats is not None and "batch_mean" in rec:
                stats.append((rec["batch_mean"], rec["batch_var"]))
        return cur


class _CostNetTrain(torch.autograd.Function):
    """pred_ind = soft arg-max of CostNet(cost volume) in training mode, differentiable in CostNet's weights and biases."""

    @staticmethod
    def forward(ctx, net, equi_s, equi_t, stats, *params):
        ind, saved = net._forward_train(equi_s, equi_t, stats)
        ctx.net, ctx.saved = net, saved
        return ind

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        grads = ctx.net._backward_train(ctx.saved, g.double().contiguous())
        return (None, None, None, None) + tuple(grads)


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
        self.force_tf32 = False
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
        for i, l in enumerate(L):
            kd, kh, kw = l["k"]
            OD, OH, OW = D - kd + 1, H - kh + 1, W - kw + 1
            if use_sd and l.get("w_sd") is not None and H == 1 and cur is not None:
                nxt = L[i + 1] if i + 1 < len(L) else None
                nxt_sd = nxt is not None and nxt.get("w_sd") is not None
                out = (ops.conv_sd_buffer(maxM, l["cout"], dev, OD * OW) if nxt_sd
                       else torch.empty((maxM, l["cout"] // 4, OD * OW, 4), dtype=torch.float32, device=dev))
                ops.conv_layer_sd(ops.GEOM_VALID3D, cur, l["w_sd"], l["b"], out, maxM, l["cin"], l["cout"], l["relu"], flag, d_n=d_M, D=D, W=W)
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

    def train_params(self):
        """(weight, bias) of every convolution, in layer order: the inputs the training Function differentiates."""
        return [t for (ci, _, _) in self.layers for t in (self.ops[ci].weight, self.ops[ci].bias)]

    def forward_train(self, equi_s, equi_t, stats=None):
        """Training mode, patch i of equi_s against patch i of equi_t ([M,32,7,20] full maps; rows 1..ele_n-2 enter the
        cost volume) -> pred_ind [M] (reference CostVolume.forward, models/BUFFERX.py:52-69), carrying a grad_fn when
        gradients are enabled and a convolution parameter requires them.  Each BatchNorm normalises with the batch
        statistics over M x its output positions and updates its running statistics once."""
        return _CostNetTrain.apply(self, equi_s.contiguous(), equi_t.contiguous(), stats, *self.train_params())

    def _forward_train(self, equi_s, equi_t, stats):
        M = equi_s.shape[0]
        cur = ops.costvol(equi_s, equi_t)                 # float64 [M, 8, 20*5*20, 4]
        D, H, W = 20, 5, 20
        saved = []
        for i in range(len(self.layers)):
            cur, rec = self._layer_train(i, cur, M, ops.GEOM_VALID3D, D, H, W)
            D, H, W = rec["out"]
            saved.append(rec)
            if stats is not None and "batch_mean" in rec:
                stats.append((rec["batch_mean"], rec["batch_var"]))
        logits = cur.view(M, -1)
        return ops.softargmax(logits).float(), dict(layers=saved, logits=logits)

    def _backward_train(self, saved, g):
        dy = ops.softargmax(saved["logits"], g)           # dL/dlogits [M, 20] == blocked [M, 5, 1, 4]
        grads = []
        for i in reversed(range(len(self.layers))):
            rec = saved["layers"][i]
            conv = self.ops[self.layers[i][0]]
            dy = dy.view(rec["z"].shape)
            if "scale" in rec:                            # ReLU mask + batch-statistics BatchNorm backward (affine=False)
                dz, _ = ops.bn_backward(dy, rec["z"], rec["y"], rec["batch_mean"], rec["scale"], torch.ones_like(rec["scale"]))
            else:
                dz = dy
            db = ops.channel_sums(dz)[0]
            dx, dW = ops.conv_backward(rec["x"], dz, rec["Wt"], *rec["geom"], want_dx=i > 0)
            grads = [dW.permute(2, 1, 0).reshape(conv.weight.shape).to(conv.weight.dtype), db.to(conv.bias.dtype)] + grads
            dy = dx
        return grads
