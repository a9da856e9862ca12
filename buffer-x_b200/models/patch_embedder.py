"""Mini-SpinNet patch descriptor on H100 kernels.

Mirrors ``MiniSpinNet`` of /root/reference/models/patch_embedder.py (constructor :16-42, forward :44-90,
same sub-module names -> same state_dict keys ``pnt_layer.{0,1}``, ``pool_layer.{0,1,3,4}``,
``conv_net.ops.*``).  select_patches -> axis_align -> normalize -> SPT -> pnt_layer+max -> Cylindrical_Net -> attention
pooling, every stage a hand-written CUDA kernel behind the C-ABI.  ``forward`` is the eval-mode forward; ``forward_train``
normalises every BatchNorm with its batch statistics and updates the running statistics, as the module does under
model.train() (the Pose training stage runs it with the descriptor network frozen: no gradients flow here).
``forward_desc_train`` is the Desc training stage's forward: float64 from the point layer on (bx_train_desc.cu), behind
one autograd Function whose backward gives the gradients of every MiniSpinNet parameter.
"""
import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from bufferx_b200 import ops
from . import patchnet as pn


def voxel_table(rad_n, azi_n, ele_n):
    """[rad_n*ele_n*azi_n,3] fp32 voxel centres, fp64 on the host then one cast -- the arithmetic of
    get_voxel_coordinate (/root/reference/utils/common.py:422-428; s2_grid :248-262, change_coordinates
    :392-405) for radius 1 (patch_embedder.py:70)."""
    beta = np.linspace(0, np.pi, num=ele_n, endpoint=False) + np.pi / ele_n / 2
    alpha = np.linspace(0, 2 * np.pi, num=azi_n, endpoint=False) + np.pi / azi_n
    Bm, Am = np.meshgrid(beta, alpha, indexing="ij")
    Bm, Am = Bm.flatten(), Am.flatten()
    s2 = np.stack([np.sin(Bm) * np.cos(Am), np.sin(Bm) * np.sin(Am), np.cos(Bm)], axis=1)
    shells = (np.arange(rad_n) / rad_n + 1 / (2 * rad_n)).reshape(rad_n, 1, 1)
    return (shells * s2[None]).reshape(-1, 3).astype(np.float32)


def derotation_table(azi_n):
    """(cos, sin) of -a*2pi/azi_n, fp64 then fp32 (var_to_invar, utils/common.py:483-491)."""
    ang = -1.0 * np.arange(azi_n) * (2 * np.pi / azi_n)
    return np.stack([np.cos(ang), np.sin(ang)], axis=1).astype(np.float32)


def pnt_stats_from_moments(mo, Wp, bp):
    """Batch mean and biased variance of the linear point layer y = Wp x + bp over R samples, from the float64 moments
    mo [9] / R of its inputs (E[x], E[y], E[z], E[xx], E[xy], E[xz], E[yy], E[yz], E[zz], as ops.moments3 orders them):
    mean = Wp E[x] + bp, var = diag(Wp Cov(x) Wp^T), Cov(x) = E[x x^T] - E[x] E[x]^T (clamped at 0)."""
    Ex = mo[:3]
    Exx = torch.stack([mo[[3, 4, 5]], mo[[4, 6, 7]], mo[[5, 7, 8]]])
    cov = Exx - Ex[:, None] * Ex[None, :]
    mean = Wp @ Ex + bp
    var = torch.clamp(((Wp @ cov) * Wp).sum(dim=1), min=0.0)
    return mean, var


class _DescTrain(torch.autograd.Function):
    """(desc, equi) of MiniSpinNet in training mode from the de-rotated point-layer inputs, differentiable in its parameters."""

    @staticmethod
    def forward(ctx, net, inv, stats, *params):
        desc, equi, saved = net._desc_forward_train(inv, stats)
        ctx.net, ctx.saved = net, saved
        return desc, equi

    @staticmethod
    @once_differentiable
    def backward(ctx, ddesc, dequi):
        grads = ctx.net._desc_backward_train(ctx.saved, ddesc, dequi)
        return (None, None, None) + tuple(g if need else None for g, need in zip(grads, ctx.needs_input_grad[3:]))


class MiniSpinNet(nn.Module):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.patch_sample = config.patch.num_points_per_patch
        self.rad_n = config.patch.rad_n
        self.azi_n = config.patch.azi_n
        self.ele_n = config.patch.ele_n
        self.delta = config.patch.delta
        self.voxel_sample = config.patch.voxel_sample
        self.pnt_layer = nn.Sequential(nn.Conv2d(3, 16, kernel_size=(1, 1)), nn.BatchNorm2d(16), nn.ReLU(True))
        self.pool_layer = nn.Sequential(nn.Conv2d(32, 16, kernel_size=(1, 1)), nn.BatchNorm2d(16), nn.ReLU(True),
                                        nn.Conv2d(16, 1, kernel_size=(1, 1)), nn.BatchNorm2d(1), nn.ReLU(True))
        self.conv_net = pn.Cylindrical_Net(inchan=16, dim=32)
        self._prep = None
        self._prep_key = None

    # ---- folded small layers + geometry tables, cached per device -------------------------------------
    def _apply(self, fn, *a, **k):
        self._prep = None
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self._prep = None
        return super()._load_from_state_dict(*a, **k)

    def prepared(self, device):
        key = pn.state_version(self.pnt_layer) + pn.state_version(self.pool_layer)
        if self._prep is None or self._prep["device"] != device or self._prep_key != key:
            self._prep_key = key
            bn = self.pnt_layer[1]
            Wt, b = pn.fold_conv_bn(self.pnt_layer[0].weight, self.pnt_layer[0].bias, bn.running_mean, bn.running_var,
                                    bn.weight, bn.bias, bn.eps)          # [1,3,16]
            w_pnt = Wt[0].t().contiguous()                                 # [16,3]
            b1n, b2n = self.pool_layer[1], self.pool_layer[4]
            W1, b1 = pn.fold_conv_bn(self.pool_layer[0].weight, self.pool_layer[0].bias, b1n.running_mean, b1n.running_var,
                                     b1n.weight, b1n.bias, b1n.eps)        # [1,32,16]
            W2, b2 = pn.fold_conv_bn(self.pool_layer[3].weight, self.pool_layer[3].bias, b2n.running_mean, b2n.running_var,
                                     b2n.weight, b2n.bias, b2n.eps)        # [1,16,1]
            self._prep = dict(
                device=device,
                w_pnt=w_pnt.to(device), b_pnt=b.to(device),
                w1=W1[0].contiguous().to(device), b1=b1.to(device),
                w2=W2[0, :, 0].contiguous().to(device), b2=b2.to(device),
                voxels=torch.from_numpy(voxel_table(self.rad_n, self.azi_n, self.ele_n)).to(device),
                rot=torch.from_numpy(derotation_table(self.azi_n)).to(device),
            )
        return self._prep

    def _front(self, pts, kpts, des_r, is_aligned_to_global_z, is_aug, perm, aug_angles, want_idx=False):
        """The front end every forward shares (patch_embedder.py:44-67): the permutation, patch selection, local reference
        frames and, with ``is_aug``, the SO(2) augmentation -> (prep, patches, idx, delta, R, rand_axis, aug_R)."""
        pts = pts[0].contiguous()
        kpts = kpts[0].contiguous()
        dev = pts.device
        N = pts.shape[0]
        if perm is None:
            # the reference consumes NumPy's GLOBAL RNG here, once per call: keep that coupling
            perm = np.random.choice(N, N, replace=False)
        if not isinstance(perm, torch.Tensor):
            perm = torch.from_numpy(np.ascontiguousarray(perm, dtype=np.int32)).to(dev, non_blocking=True)
        prep = self.prepared(dev)
        pts4 = ops.permute_cloud(pts, perm)
        patches, idx = ops.select_patches(pts4, kpts, des_r, self.patch_sample, want_idx=want_idx)
        delta, R, rand_axis = ops.lrf(patches, des_r, bool(is_aligned_to_global_z))
        aug_R = None
        if is_aug:
            if aug_angles is None:
                # the reference draws angles = r * 2 * pi in fp64 (after the permutation) and casts them to fp32
                aug_angles = (np.random.random([kpts.shape[0], 1]) * 2 * np.pi)[:, 0].astype(np.float32)
            ang = torch.as_tensor(np.ascontiguousarray(aug_angles, dtype=np.float32)).to(dev, non_blocking=True)
            aug_R = ops.so2_augment(delta, rand_axis, ang)
        return prep, patches, idx, delta, R, rand_axis, aug_R

    def _pnt_batch_stats(self, inv, stats):
        """The point layer's batch statistics over every sample of inv [..., 3] (zero slots included) from the float64
        moments of its inputs (it is linear: mean = W E[x] + b, var = diag(W Cov(x) W^T)); updates its running statistics
        once and appends (mean, var) to ``stats`` -> (mean, var, W [16, 3], b [16] float64, moments [9])."""
        conv, bn = self.pnt_layer[0], self.pnt_layer[1]
        R_n = inv.numel() // 3
        mo = ops.moments3(inv)
        Wp = conv.weight.detach().double().view(16, 3).contiguous()
        bp = conv.bias.detach().double().contiguous()
        mean, var = pnt_stats_from_moments(mo / R_n, Wp, bp)
        pn.bn_batch_stats(torch.stack([mean * R_n, (var + mean * mean) * R_n]), R_n, bn)
        if stats is not None:
            stats.append((mean, var))
        return mean, var, Wp, bp, mo

    def forward(self, pts, kpts, des_r, is_aligned_to_global_z, z_axis=None, is_aug=False, perm=None, debug=False, aug_angles=None):
        """pts [1,N,3], kpts [1,K,3] CUDA f32; des_r python float or 1-element CUDA tensor.
        ``perm`` (optional int32 [N]) replaces the host draw of the reference (patch_embedder.py:96).
        ``is_aug``: SO(2) augmentation of the normalised patches and rand_axis (patch_embedder.py:54-67), one z-rotation per
        patch; the angles are drawn from NumPy's global RNG after the permutation, like the reference, unless ``aug_angles``
        ([K] fp32) are given.  ``aug_rotation`` is then the [K,3,3] rotations (None without augmentation)."""
        if z_axis is not None:
            raise NotImplementedError("an externally supplied z_axis is a training-time option outside the forward built here")
        prep, patches, idx, delta, R, rand_axis, aug_R = self._front(pts, kpts, des_r, is_aligned_to_global_z, is_aug, perm, aug_angles,
                                                                     want_idx=debug)
        res = ops.spt_pnt(delta, prep["voxels"], prep["rot"], self.delta / self.rad_n, self.voxel_sample, prep["w_pnt"],
                          prep["b_pnt"], self.azi_n, debug=debug)
        feat = res[0] if debug else res                                  # [K,4,V,4] channel-blocked
        K = delta.shape[0]
        x, _ = self.conv_net(feat)                                       # [K,8,140,4] channel-blocked
        desc, equi = ops.pool_desc(x, prep["w1"], prep["b1"], prep["w2"], prep["b2"], channels_last=True)
        out = {"desc": desc, "equi": equi, "rand_axis": rand_axis, "R": R, "patches": delta, "aug_rotation": aug_R}
        if debug:
            out.update(idx=idx, raw_patches=patches, vidx=res[1], inv=res[2], feat=ops.from_blocked(feat),
                       x=ops.from_blocked(x).view(K, -1, self.ele_n, self.azi_n))
        return out

    def forward_train(self, pts, kpts, des_r, is_aligned_to_global_z, is_aug=False, perm=None, aug_angles=None, stats=None):
        """MiniSpinNet.forward under model.train() (patch_embedder.py:44-90): the same patches, frames, augmentation and SPT
        as ``forward``, but each of the ten BatchNorm layers normalises with its batch statistics and updates its running
        statistics once.  The point layer's statistics over the K x 420 x 10 samples (zero slots included) follow from the
        float64 moments of its de-rotated 3-vectors (it is linear: mean = W E[x] + b, var = diag(W Cov(x) W^T)); the pool
        layer's from its 1x1 convolutions over K x 140 positions.  ``stats``: optional list receiving (batch mean, batch
        variance) of every BatchNorm in module order (pnt_layer, conv_net, pool_layer), float64.  Returns ``forward``'s dict."""
        prep, _, _, delta, R, rand_axis, aug_R = self._front(pts, kpts, des_r, is_aligned_to_global_z, is_aug, perm, aug_angles)
        dev = delta.device
        args = (delta, prep["voxels"], prep["rot"], self.delta / self.rad_n, self.voxel_sample)
        _, _, inv = ops.spt_pnt(*args, prep["w_pnt"], prep["b_pnt"], self.azi_n, debug=True)   # the samples the point layer sees
        mean, var, _, _, _ = self._pnt_batch_stats(inv, stats)
        conv, bn = self.pnt_layer[0], self.pnt_layer[1]
        Wt, b = pn.fold_conv_bn(conv.weight, conv.bias, mean, var, bn.weight, bn.bias, bn.eps)
        feat = ops.spt_pnt(*args, Wt[0].t().contiguous().to(dev), b.to(dev), self.azi_n)
        x = self.conv_net.forward_train(feat, stats)                      # [K,8,140,4]
        # pool layer: two 1x1 convolutions, each followed by a batch-statistics BatchNorm and ReLU
        c1, b1n, c2, b2n = self.pool_layer[0], self.pool_layer[1], self.pool_layer[3], self.pool_layer[4]
        K = x.shape[0]
        W1, bb1 = pn.fold_conv_bn(c1.weight, c1.bias)                    # [1,32,16]
        z1 = ops.conv1x1(x, W1[0].contiguous(), bb1)
        m1, v1 = pn.bn_batch_stats(ops.channel_sums(z1), K * 140, b1n)
        sc, sh = pn.bn_scale_shift(m1, v1, b1n)
        h = ops.bn_apply(z1, sc, sh, True)
        W2, bb2 = pn.fold_conv_bn(c2.weight, c2.bias)                    # [1,16,1]
        w2p = torch.zeros((16, 4), dtype=torch.float32, device=dev)
        w2p[:, :1] = W2[0]
        b2p = torch.zeros(4, dtype=torch.float32, device=dev)
        b2p[:1] = bb2
        z2 = ops.conv1x1(h, w2p, b2p)                                     # channel 0 is the attention logit
        m2, v2 = pn.bn_batch_stats(ops.channel_sums(z2)[:, :1], K * 140, b2n)
        if stats is not None:
            stats += [(m1, v1), (m2, v2)]
        Wf1, bf1 = pn.fold_conv_bn(c1.weight, c1.bias, m1, v1, b1n.weight, b1n.bias, b1n.eps)
        Wf2, bf2 = pn.fold_conv_bn(c2.weight, c2.bias, m2, v2, b2n.weight, b2n.bias, b2n.eps)
        desc, equi = ops.pool_desc(x, Wf1[0].contiguous(), bf1, Wf2[0, :, 0].contiguous(), bf2, channels_last=True)
        return {"desc": desc, "equi": equi, "rand_axis": rand_axis, "R": R, "patches": delta, "aug_rotation": aug_R}

    def forward_desc_train(self, pts, kpts, des_r, is_aligned_to_global_z, perm=None, stats=None):
        """MiniSpinNet.forward of the Desc training stage (patch_embedder.py:44-90 under model.train(), no augmentation): the
        patches, frames and SPT of ``forward``, then ``train_desc``.  ``desc`` and ``equi`` carry a grad_fn into the
        parameters that require grad.  Returns ``forward``'s dict."""
        prep, _, _, delta, R, rand_axis, _ = self._front(pts, kpts, des_r, is_aligned_to_global_z, False, perm, None)
        _, _, inv = ops.spt_pnt(delta, prep["voxels"], prep["rot"], self.delta / self.rad_n, self.voxel_sample, prep["w_pnt"],
                                prep["b_pnt"], self.azi_n, debug=True)
        desc, equi = self.train_desc(inv, stats)
        return {"desc": desc, "equi": equi, "rand_axis": rand_axis, "R": R, "patches": delta, "aug_rotation": None}

    def train_desc(self, inv, stats=None):
        """Training mode from the de-rotated samples inv [K, V, nv, 3] (fp32, zero slots included) -> (desc [K, 32], equi
        [K, 32, ele_n, azi_n]) fp32, evaluated in float64.  Every BatchNorm normalises with its batch statistics and updates
        its running statistics once (also under torch.no_grad()).  ``stats``: optional list receiving (batch mean, batch
        variance) of every BatchNorm in module order (pnt_layer, conv_net, pool_layer), float64."""
        if self.rad_n * self.ele_n * self.azi_n != 420 or self.azi_n != 20 or self.rad_n != 3:
            raise ops.BufferXError("train_desc: the Desc training kernels are built for 3 x 7 x 20 cylindrical voxels")
        return _DescTrain.apply(self, inv.contiguous(), [] if stats is None else stats, *self.parameters())

    def _desc_forward_train(self, inv, stats):
        F64 = torch.float64
        dev = inv.device
        K = inv.shape[0]
        mean, var, Wp, bp, mo = self._pnt_batch_stats(inv, stats)
        bn = self.pnt_layer[1]
        scale, shift = pn.bn_scale_shift(mean, var, bn, F64)
        feat, arg = ops.pnt_forward(inv, Wp, bp, scale, shift)
        pnt = dict(inv=inv, arg=arg, W=Wp, b=bp, mean=mean.contiguous(), rstd=(1.0 / torch.sqrt(var + bn.eps)).contiguous(),
                   gamma=bn.weight.detach().double().contiguous(), scale=scale, shift=shift, mo=mo)
        # Cylindrical_Net on the fp64 tensor cores, each BatchNorm'd layer normalised with its batch statistics
        net = self.conv_net
        N = K * 140
        cur, layers = feat, []
        for i, (ci, bi, _) in enumerate(net.layers):
            c = net.ops[ci]
            Din = 3 if i == 0 else 1
            Wt = c.weight.detach().double().reshape(c.out_channels, c.in_channels, -1).permute(2, 1, 0).contiguous()
            z = ops.cyl_forward(cur, Wt, c.bias.detach().double().contiguous(), Din)
            rec = dict(x=cur, z=z, Wt=Wt, Din=Din)
            if bi is not None:
                m, v = pn.bn_batch_stats(ops.channel_sums(z), N, net.ops[bi])
                sc, sh = pn.bn_scale_shift(m, v, net.ops[bi], F64)
                stats.append((m, v))
                cur = ops.bn_apply(z, sc, sh, True)
                rec.update(mean=m, scale=sc, y=cur)
            else:
                cur = z
            layers.append(rec)
        x = cur
        # pool layer: two 1x1 convolutions with affine batch-statistics BatchNorm and ReLU -> attention w; pooling
        c1, b1n, c2, b2n = self.pool_layer[0], self.pool_layer[1], self.pool_layer[3], self.pool_layer[4]
        W1 = c1.weight.detach().double().view(16, 32).t().contiguous()                    # [32, 16]
        z1 = ops.conv1x1(x, W1, c1.bias.detach().double().contiguous())
        m1, v1 = pn.bn_batch_stats(ops.channel_sums(z1), N, b1n)
        sc1, sh1 = pn.bn_scale_shift(m1, v1, b1n, F64)
        h = ops.bn_apply(z1, sc1, sh1, True)
        W2 = torch.zeros((16, 4), dtype=F64, device=dev)                                   # one output channel, padded to 4
        W2[:, 0] = c2.weight.detach().double().view(16)
        b2 = torch.zeros(4, dtype=F64, device=dev)
        b2[0] = c2.bias.detach().double()[0]
        z2 = ops.conv1x1(h, W2, b2)
        m2, v2 = pn.bn_batch_stats(ops.channel_sums(z2)[:, :1], N, b2n)
        sc2, sh2 = pn.bn_scale_shift(m2, v2, b2n, F64)

        def pad(t):                      # the one attention channel, padded to the 4 of a blocked image
            return torch.cat([t.reshape(1).double(), torch.zeros(3, dtype=F64, device=dev)])
        w = ops.bn_apply(z2, pad(sc2), pad(sh2), True)
        stats += [(m1, v1), (m2, v2)]
        f, desc, equi = ops.pool_forward(x, w)
        pool = dict(x=x, z1=z1, h=h, z2=z2, w=w, f=f, W1=W1, W2=W2,
                    bn1=(m1.contiguous(), (1.0 / torch.sqrt(v1 + b1n.eps)).contiguous(), b1n.weight.detach().double().contiguous()),
                    bn2=tuple(pad(t) for t in (m2, 1.0 / torch.sqrt(v2 + b2n.eps), b2n.weight.detach())))
        return desc, equi.view(K, 32, self.ele_n, self.azi_n), dict(pnt=pnt, layers=layers, pool=pool, K=K)

    def _desc_backward_train(self, saved, ddesc, dequi):
        """The gradients of every parameter (in self.parameters() order) from dL/ddesc, dL/dequi (either may be None)."""
        K = saved["K"]
        dev = saved["pool"]["x"].device
        ddesc = torch.zeros((K, 32), dtype=torch.float32, device=dev) if ddesc is None else ddesc.float().contiguous()
        dequi = torch.zeros((K, 32, self.ele_n, self.azi_n), dtype=torch.float32, device=dev) if dequi is None else dequi.float().contiguous()
        g = {}
        P = saved["pool"]
        dx, dw = ops.pool_backward(P["x"], P["w"], P["f"], ddesc, dequi)
        dz2, s2 = ops.bn_backward(dw, P["z2"], P["w"], *P["bn2"])        # masked by the forward's ReLU output
        g["pool_layer.4.weight"], g["pool_layer.4.bias"] = s2[1, :1], s2[0, :1]
        g["pool_layer.3.weight"] = ops.cross_sums(P["h"], dz2)[:, :1].t()
        g["pool_layer.3.bias"] = ops.channel_sums(dz2)[0, :1]
        dh = ops.conv1x1(dz2, P["W2"].t().contiguous())
        dz1, s1 = ops.bn_backward(dh, P["z1"], P["h"], *P["bn1"])
        g["pool_layer.1.weight"], g["pool_layer.1.bias"] = s1[1], s1[0]
        g["pool_layer.0.weight"] = ops.cross_sums(P["x"], dz1).t()
        g["pool_layer.0.bias"] = ops.channel_sums(dz1)[0]
        dy = ops.conv1x1(dz1, P["W1"].t().contiguous(), out=dx)
        net = self.conv_net
        for i in reversed(range(len(net.layers))):
            rec = saved["layers"][i]
            if "scale" in rec:                        # ReLU mask + batch-statistics BatchNorm backward (affine=False)
                dz, _ = ops.bn_backward(dy, rec["z"], rec["y"], rec["mean"], rec["scale"], torch.ones_like(rec["scale"]))
            else:
                dz = dy
            ci = net.layers[i][0]
            g[f"conv_net.ops.{ci}.bias"] = ops.channel_sums(dz)[0]
            dy, dW = ops.cyl_backward(rec["x"], dz, rec["Wt"], rec["Din"])
            g[f"conv_net.ops.{ci}.weight"] = dW.permute(2, 1, 0)
        Q = saved["pnt"]
        o = ops.pnt_backward(Q["inv"], Q["arg"], dy, Q["W"], Q["b"], Q["mean"], Q["rstd"], Q["gamma"], Q["scale"], Q["shift"], Q["mo"])
        g["pnt_layer.0.weight"], g["pnt_layer.0.bias"] = o[:, :3], o[:, 3]
        g["pnt_layer.1.weight"], g["pnt_layer.1.bias"] = o[:, 4], o[:, 5]
        return [g[name].reshape(p.shape).to(p.dtype).contiguous() for name, p in self.named_parameters()]

    def forward_multi(self, jobs, is_aligned_to_global_z, radii=None, counts=None, npts=None):
        """Descriptors of several (cloud, key-points, radius, permutation) jobs in ONE pass through SPT, the
        convolution stack and the pooling layer (all CTA-per-patch kernels: batching the 2 x num_scales calls of a
        pair removes five of six launch tails and wave-quantisation losses).  Per-job results are views into the
        batched buffers; same arithmetic as ``forward`` per patch.  jobs: list of (pts [N,3], kpts [K,3], des_r
        1-element CUDA tensor, perm int32 [N]).
        ``counts`` (early-exit pairs: the later scales' work sized on the device, see BufferX._enqueue_device_exit): a dict of
        int32 CUDA tensors, "job" [1] = key-points of every job, "group" [len(radii)] = patches of every radius group, "total" [1]
        = patches of the batch (jobs of equal size, (src, tgt) per radius).  Patches beyond them are not computed and their
        result rows are undefined.
        ``npts`` (size-class slots, see BufferX.enable_cuda_graphs): one 1-element int32 CUDA tensor per job, the points of its
        cloud; pts and perm are then capacity buffers whose first npts[j] entries hold the cloud and its permutation, and the
        scan / hash-grid choice follows the capacity.  Results are those of the exact clouds."""
        dev = jobs[0][0].device
        prep = self.prepared(dev)
        P = self.patch_sample
        Ks = [j[1].shape[0] for j in jobs]
        Kt = sum(Ks)
        patches = torch.empty((Kt, P, 3), dtype=torch.float32, device=dev)
        delta = torch.empty_like(patches)
        R_all = torch.empty((Kt, 3, 3), dtype=torch.float32, device=dev)
        ra_all = torch.empty((Kt, 3), dtype=torch.float32, device=dev)
        Rs, axes = [], []
        o = 0
        # `radii` = the contiguous device array of per-scale radii when the jobs are (src, tgt) per scale with equal key-point
        # counts: the local reference frames of all jobs then run in ONE launch (patch k uses radii[k // (2 K)])
        one_lrf = radii is not None and len(set(Ks)) == 1 and len(jobs) == 2 * radii.numel()
        one_sel = len(jobs) <= 16 and all(isinstance(j[2], torch.Tensor) for j in jobs)   # all patch gatherings of the pair in one launch
        if counts is not None and not (one_lrf and one_sel):
            raise ops.BufferXError("forward_multi: device-side counts need equal-size (src, tgt) jobs per radius and device radii")
        if npts is not None and not one_sel:
            raise ops.BufferXError("forward_multi: device-side point counts need device radii and at most 16 jobs")
        sel = []
        for j, ((pts, kpts, des_r, perm), K) in enumerate(zip(jobs, Ks)):
            sel.append((ops.permute_cloud(pts.contiguous(), perm, d_N=None if npts is None else npts[j]), kpts.contiguous(), des_r))
            Rs.append(R_all[o:o + K])
            axes.append(ra_all[o:o + K])
            o += K
        # small clouds: all jobs through the streaming scan in one launch; larger ones: all jobs through the hash grid, one launch
        # per phase; a mix of both (C5: 60 k vs 30 k points is above the threshold on both sides; 5 k vs 20 k would not be): job by job
        big = [pts4.shape[0] >= ops.GRID_MIN_POINTS for (pts4, _, _) in sel]
        job_cnt = None if counts is None else [counts["job"]] * len(jobs)
        if one_sel and (all(big) or not any(big)):
            ops.select_patches_batched(sel, P, patches, grid=all(big), d_K=job_cnt, d_N=npts)
        o = 0
        for j, ((pts4, kpts, des_r), K) in enumerate(zip(sel, Ks)):
            if not (one_sel and (all(big) or not any(big))):
                if counts is not None or npts is not None:      # job by job, each with its device counts
                    ops.select_patches_batched([(pts4, kpts, des_r)], P, patches[o:o + K], grid=big[j],
                                               d_K=None if job_cnt is None else job_cnt[:1], d_N=None if npts is None else npts[j:j + 1])
                elif big[j] and isinstance(des_r, torch.Tensor):
                    ops.select_patches_grid(pts4, kpts, des_r, P, patches=patches[o:o + K])
                else:
                    ops.select_patches(pts4, kpts, des_r, P, patches=patches[o:o + K])
            if not one_lrf:
                ops.lrf(patches[o:o + K], des_r, bool(is_aligned_to_global_z), delta=delta[o:o + K], Rt=R_all[o:o + K], ra=ra_all[o:o + K])
            o += K
        if one_lrf:
            ops.lrf(patches, radii, bool(is_aligned_to_global_z), delta=delta, Rt=R_all, ra=ra_all, r_group=2 * Ks[0],
                    d_K=None if counts is None else counts["group"])
        net = self.conv_net
        if not net.force_tf32 and self.rad_n * self.ele_n * self.azi_n == 420 and self.azi_n == 20:
            # production: features straight into the presplit fp16 format the first conv layer fetches with bulk copies
            feat = ops.spt_pnt_sd(delta, prep["voxels"], prep["rot"], self.delta / self.rad_n, self.voxel_sample, prep["w_pnt"],
                                  prep["b_pnt"], self.azi_n, net.overflow_flag(dev), d_K=None if counts is None else counts["total"])
        else:
            feat = ops.spt_pnt(delta, prep["voxels"], prep["rot"], self.delta / self.rad_n, self.voxel_sample, prep["w_pnt"],
                               prep["b_pnt"], self.azi_n)
        total = None if counts is None else counts["total"]
        x, _ = self.conv_net(feat, K=Kt, d_n=total)
        desc, equi = ops.pool_desc(x, prep["w1"], prep["b1"], prep["w2"], prep["b2"], channels_last=True, d_K=total)
        outs, o = [], 0
        for K, R, ra in zip(Ks, Rs, axes):
            outs.append({"desc": desc[o:o + K], "equi": equi[o:o + K], "rand_axis": ra, "R": R, "patches": delta[o:o + K],
                         "aug_rotation": None})
            o += K
        self.last_multi = {"desc": desc, "equi": equi, "R": R_all}       # the batched buffers behind the per-job views
        return outs

    def get_parameter(self):
        return list(self.parameters())
