"""Mini-SpinNet patch descriptor on H100 kernels.

Mirrors ``MiniSpinNet`` of /root/reference/models/patch_embedder.py (constructor :16-42, forward :44-90,
same sub-module names -> same state_dict keys ``pnt_layer.{0,1}``, ``pool_layer.{0,1,3,4}``,
``conv_net.ops.*``).  Eval mode only: select_patches -> axis_align -> normalize -> SPT -> pnt_layer+max ->
Cylindrical_Net -> attention pooling, every stage a hand-written CUDA kernel behind the C-ABI.
"""
import numpy as np
import torch
import torch.nn as nn

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

    # ---- folded small layers + geometry tables, cached per device -------------------------------------
    def _apply(self, fn, *a, **k):
        self._prep = None
        return super()._apply(fn, *a, **k)

    def _load_from_state_dict(self, *a, **k):
        self._prep = None
        return super()._load_from_state_dict(*a, **k)

    def prepared(self, device):
        if self._prep is None or self._prep["device"] != device:
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

    def forward(self, pts, kpts, des_r, is_aligned_to_global_z, z_axis=None, is_aug=False, perm=None, debug=False, aug_angles=None):
        """pts [1,N,3], kpts [1,K,3] CUDA f32; des_r python float or 1-element CUDA tensor.
        ``perm`` (optional int32 [N]) replaces the host draw of the reference (patch_embedder.py:96).
        ``is_aug``: SO(2) augmentation of the normalised patches and rand_axis (patch_embedder.py:54-67), one z-rotation per
        patch; the angles are drawn from NumPy's global RNG after the permutation, like the reference, unless ``aug_angles``
        ([K] fp32) are given.  ``aug_rotation`` is then the [K,3,3] rotations (None without augmentation)."""
        if z_axis is not None:
            raise NotImplementedError("an externally supplied z_axis is a training-time option outside the forward built here")
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
        patches, idx = ops.select_patches(pts4, kpts, des_r, self.patch_sample, want_idx=debug)
        delta, R, rand_axis = ops.lrf(patches, des_r, bool(is_aligned_to_global_z))
        aug_R = None
        if is_aug:
            if aug_angles is None:
                # the reference draws angles = r * 2 * pi in fp64 and casts them to fp32
                aug_angles = (np.random.random([kpts.shape[0], 1]) * 2 * np.pi)[:, 0].astype(np.float32)
            ang = torch.as_tensor(np.ascontiguousarray(aug_angles, dtype=np.float32)).to(dev, non_blocking=True)
            aug_R = ops.so2_augment(delta, rand_axis, ang)
        res = ops.spt_pnt(delta, prep["voxels"], prep["rot"], self.delta / self.rad_n, self.voxel_sample, prep["w_pnt"],
                          prep["b_pnt"], self.azi_n, debug=debug)
        feat = res[0] if debug else res                                  # [K,4,V,4] channel-blocked
        K = kpts.shape[0]
        x, _ = self.conv_net(feat)                                       # [K,8,140,4] channel-blocked
        desc, equi = ops.pool_desc(x, prep["w1"], prep["b1"], prep["w2"], prep["b2"], channels_last=True)
        out = {"desc": desc, "equi": equi, "rand_axis": rand_axis, "R": R, "patches": delta, "aug_rotation": aug_R}
        if debug:
            out.update(idx=idx, raw_patches=patches, vidx=res[1], inv=res[2], feat=ops.from_blocked(feat),
                       x=ops.from_blocked(x).view(K, -1, self.ele_n, self.azi_n))
        return out

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
